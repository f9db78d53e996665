"""Cost of the training loop's additions on the GPU, in one process.

    python tools/bench_training_loop.py [--steps 8] [--warmup 2] [--valid 64] [--search 32]

  * train: bench.py's `--mode train` step (B=64 x T=1500, WSJ architecture, L=190, StepClipping + momentum + AdaDelta +
    max-norm) with adaptive clipping on and off, two recognizers with the same parameters, process_batch timed with
    CUDA events and a synchronisation per step, the two alternating step by step; medians, minima and kernel launches
    per step (lvsr_launch_count) of each.
  * valid: a TIMIT-shaped validation pass (3 x BiGRU(256), 123 features, location attention, V=63, T=400, L=50, batches
    of 64 as nips_baseline's validation_batch_size): SpeechRecognizer.validation_statistics (cost + alignment
    statistics) in utterances/s, and the alignment-statistics kernel alone in ms per batch.
  * per: the PER monitor's beam search (beam 10) over `--search` utterances of that shape, through beam_search_many in
    one call against one beam_search per utterance, in utterances/s.
One JSON object with the card's name and power limit.  Writes nothing.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit (--steps 6 --warmup 2, one call): train 135.4 ms per
step with the fixed threshold, 135.9 ms with adaptive clipping (medians of 6; 1505 launches per step each); validation
6340 utterances/s, of which the statistics kernel takes 0.081 ms per batch of 64; PER search 163 utterances/s batched
against 16.3 per utterance, the same best hypothesis for all 32.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

TIMIT = dict(num_features=123, dims_bidir=[256, 256, 256], subsample=[1, 1, 1], dim_dec=256, dim_matcher=256,
             conv_n=100, conv_num_filters=10, num_phonemes=63, post_merge_dims=[256], maxout_pieces=2)
TIMIT_BATCH = dict(B=64, T=400, F=123, L=50, V=63)


def make(pkg, dev, net, attention_type="content_and_conv"):
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": net["num_features"]}, input_num_chars={}, eos_label=net["num_phonemes"] - 1,
        num_phonemes=net["num_phonemes"], dim_dec=net["dim_dec"], dims_bidir=net["dims_bidir"],
        subsample=net["subsample"], conv_n=net["conv_n"], conv_num_filters=net["conv_num_filters"],
        dim_matcher=net["dim_matcher"], post_merge_dims=net["post_merge_dims"], post_merge_activation=pkg.Maxout(2),
        attention_type=attention_type, enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent,
        device=dev)
    rec.set_parameter_values(bench.init_values(rec.parameter_shapes()))
    return rec


def median(v):
    return sorted(v)[len(v) // 2]


def train(pkg, torch, lib, dev, steps, warmup):
    W = bench.TRAIN_WORKLOAD
    net = dict(bench.NET, num_features=W["F"], num_phonemes=W["V"])
    algos = {}
    for k in ("fixed", "adaptive"):
        rule = pkg.step_rule_from_config(bench.TRAIN_CONF, dict(max_norm=1.0))
        if k == "adaptive":
            pkg.adaptive_clipping(rule, burnin_period=500, decay_rate=0.998)
        algos[k] = pkg.GradientDescent(recognizer=make(pkg, dev, net), step_rule=rule)
        algos[k].initialize()
    x, m, labels, lm = bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"], seed=4321)
    batch = dict(zip(pkg.GradientDescent.SOURCES, (torch.as_tensor(a, device=dev) for a in (x, m, labels, lm))))
    for _ in range(max(2, warmup)):
        for a in algos.values():
            a.process_batch(batch)
    torch.cuda.synchronize(dev)
    ms = {k: [] for k in algos}
    launches = {k: [] for k in algos}
    for _ in range(steps):
        for k, a in algos.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            lib.lvsr_launch_count(1)
            e0.record()
            a.process_batch(batch)
            e1.record()
            launches[k].append(int(lib.lvsr_launch_count(0)))
            torch.cuda.synchronize(dev)
            ms[k].append(e0.elapsed_time(e1))
    clip = pkg.clipping_rule(algos["adaptive"].step_rule)
    out = {"workload": W}
    for k in algos:
        out[k] = {"ms_per_step": round(median(ms[k]), 3), "ms_per_step_min": round(min(ms[k]), 3),
                  "launches_per_step": median(launches[k])}
    out["adaptive"]["next_threshold"] = clip.current_threshold()
    out["adaptive_over_fixed"] = round(out["adaptive"]["ms_per_step"] / out["fixed"]["ms_per_step"], 4)
    return out


def valid(pkg, torch, dev, rec, batches, steps):
    W = TIMIT_BATCH
    data = [bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"], seed=500 + i) for i in range(batches)]
    for b in data[:1]:
        rec.validation_statistics(*b)
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for b in data:
        rec.validation_statistics(*b)
    e1.record()
    torch.cuda.synchronize(dev)
    total_ms = e0.elapsed_time(e1)
    # the statistics kernel alone, on the weights of one batch
    x, m, labels, lm = data[0]
    att, attm = rec.encode(x, m)
    w = rec.cost_matrix(labels, lm, att, attm, return_all=True)["weights"]
    lmd = torch.as_tensor(lm, device=dev)
    out = torch.zeros((2,), dtype=torch.float64, device=dev)
    rec.alignment_statistics(w, lmd, out)
    torch.cuda.synchronize(dev)
    e0.record()
    for _ in range(steps):
        rec.alignment_statistics(w, lmd, out)
    e1.record()
    torch.cuda.synchronize(dev)
    stats_ms = e0.elapsed_time(e1) / steps
    L, B, Tp = w.shape
    return {"workload": dict(W, batches=batches), "utterances_per_s": round(batches * W["B"] / (total_ms * 1e-3), 1),
            "ms_per_batch": round(total_ms / batches, 3), "stats_kernel_ms_per_batch": round(stats_ms, 4),
            "stats_kernel_bytes_per_s": round(L * B * Tp * 4 / (stats_ms * 1e-3))}


def per(torch, dev, rec, n):
    W = TIMIT_BATCH
    x, m, _, _ = bench.synthetic_batch(n, W["T"], W["F"], W["L"], W["V"], seed=77)
    lens = m.sum(axis=0).astype(int)
    utts = [{"recordings": x[:lens[u], u]} for u in range(n)]
    rec.init_beam_search(10)
    rec.beam_search_many(utts[:2], raise_on_failure=False)
    torch.cuda.synchronize(dev)
    import time
    t0 = time.time()
    many = rec.beam_search_many(utts, raise_on_failure=False)
    t_many = time.time() - t0
    t0 = time.time()
    same = 0
    for u, r in zip(utts, many):
        try:
            outputs, _ = rec.beam_search(u)
        except pkg_error():
            outputs = None
        same += int((r is None and outputs is None) or (r is not None and outputs is not None and
                                                         list(r[0][0]) == list(outputs[0])))
    t_one = time.time() - t0
    return {"utterances": n, "beam": 10, "batched_utterances_per_s": round(n / t_many, 2),
            "per_utterance_utterances_per_s": round(n / t_one, 2), "speedup": round(t_one / t_many, 2),
            "same_best_hypothesis": same}


def pkg_error():
    import __graft_entry__ as graft
    return graft.load_package().CandidateNotFoundError


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--valid", type=int, default=6, help="validation batches of 64")
    ap.add_argument("--search", type=int, default=32, help="utterances decoded for the PER comparison")
    ap.add_argument("--only", default=None, help="comma-separated parts: train,valid,per")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_training_loop: needs a CUDA device")
    import __graft_entry__ as graft
    pkg = graft.load_package()
    lib = pkg._lib.load()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    parts = args.only.split(",") if args.only else ["train", "valid", "per"]
    out = {"gpu": bench.gpu_identity(0)}
    if "train" in parts:
        out["train"] = train(pkg, torch, lib, dev, args.steps, args.warmup)
    if "valid" in parts or "per" in parts:
        rec = make(pkg, dev, TIMIT)
        if "valid" in parts:
            out["valid"] = valid(pkg, torch, dev, rec, args.valid, args.steps)
        if "per" in parts:
            out["per"] = per(torch, dev, rec, args.search)
    print(json.dumps(out))


if __name__ == "__main__":
    np.seterr(all="ignore")
    main()
