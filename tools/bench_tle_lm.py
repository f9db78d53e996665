"""Task loss estimation with and without shallow fusion of an FST language model, on the GPU, alternating the models
in one process.

    python tools/bench_tle_lm.py [--steps 3] [--warmup 1]

The model has the TIMIT iclr_reward shape (123 features, 3 x BiGRU(256) without subsampling, 63 phonemes, Maxout(2)
readout); the LM is tests/lm_oracle.py's seeded character trigram with backoff over the 63 symbols, written as an
OpenFST vector file to a temporary directory and loaded through SpeechRecognizer(lm=...) with decode_tle.sh's
weight 0.15 (every other option at the recognizer's default).  Prints one JSON line:
  * search: lvsr_beam_search_many over 8 utterances of <= 300 frames (max_decoded_length_scale 3) at beam 10 and 200,
    for mse_gain and mse_reward, with and without the LM: milliseconds per batch (median over --steps, host clock
    around a synchronised call) and the relative cost of fusion;
  * cost_matrix: the teacher-forced cost at B=64 x T=800, L=101 for both criteria with and without the LM
    (CUDA events, median), and the relative cost of fusion;
  * gpu: card name, power limit and maximum SM clock, which every number depends on.
Synthetic inputs and parameters from fixed seeds; nothing is written to the tree.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
import lm_oracle as LO  # noqa: E402

ICLR = dict(num_features=123, dims_bidir=[256, 256, 256], subsample=[1, 1, 1], dim_dec=256, dim_matcher=512,
            conv_n=100, conv_num_filters=10, num_phonemes=63, post_merge_dims=[256])
CRITERIA = ("mse_gain", "mse_reward")
SCALE = 3.0


def make(pkg, dev, criterion, lm, cmap):
    net = ICLR
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": net["num_features"]}, input_num_chars={}, eos_label=net["num_phonemes"] - 1,
        num_phonemes=net["num_phonemes"], dim_dec=net["dim_dec"], dims_bidir=net["dims_bidir"],
        subsample=net["subsample"], conv_n=net["conv_n"], conv_num_filters=net["conv_num_filters"],
        dim_matcher=net["dim_matcher"], post_merge_dims=net["post_merge_dims"], post_merge_activation=pkg.Maxout(2),
        criterion=dict(name=criterion, min_reward=-5.0), max_decoded_length_scale=SCALE, data_prepend_eos=False,
        enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent, device=dev, lm=lm,
        character_map=cmap if lm else None)
    rec.set_parameter_values(bench.init_values(rec.parameter_shapes()))
    return rec


def median(v):
    return sorted(v)[len(v) // 2]


def time_search(torch, dev, recs, inputs, beam, steps, warmup):
    for rec in recs.values():
        rec.init_beam_search(beam)
    res = {}
    for _ in range(warmup):
        for k, rec in recs.items():
            res[k] = rec.beam_search_many(inputs, raise_on_failure=False)
    ms = {k: [] for k in recs}
    for _ in range(steps):
        for k, rec in recs.items():
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            res[k] = rec.beam_search_many(inputs, raise_on_failure=False)
            torch.cuda.synchronize(dev)
            ms[k].append((time.perf_counter() - t0) * 1e3)
    out = {}
    for k in recs:
        found = [r for r in res[k] if r is not None]
        out[k] = {"ms_per_batch_median": round(median(ms[k]), 2), "ms_per_batch_min": round(min(ms[k]), 2),
                  "decoded": len(found),
                  "mean_best_length": round(float(np.mean([len(r[0][0]) for r in found])), 1) if found else 0.0}
    for c in CRITERIA:
        out[c + "_fusion_overhead"] = round(out[c + "+lm"]["ms_per_batch_median"] /
                                            out[c]["ms_per_batch_median"] - 1.0, 4)
    return out


def time_cost(torch, dev, recs, steps, warmup):
    W = dict(B=64, T=800, F=ICLR["num_features"], L=101, V=ICLR["num_phonemes"])
    x, m, labels, lm = bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"], seed=777)   # labels end in eos
    y, ym = torch.as_tensor(labels, device=dev), torch.as_tensor(lm, device=dev)
    enc = {k: r.encode(x, m) for k, r in recs.items()}
    for _ in range(warmup):
        for k, r in recs.items():
            r.cost_matrix(y, ym, *enc[k])
    torch.cuda.synchronize(dev)
    ms = {k: [] for k in recs}
    for _ in range(steps):
        for k, r in recs.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            r.cost_matrix(y, ym, *enc[k])
            b.record()
            torch.cuda.synchronize(dev)
            ms[k].append(a.elapsed_time(b))
    out = {k: {"ms_median": round(median(v), 3), "ms_min": round(min(v), 3)} for k, v in ms.items()}
    for c in CRITERIA:
        out[c + "_fusion_overhead"] = round(out[c + "+lm"]["ms_median"] / out[c]["ms_median"] - 1.0, 4)
    out["shape"] = "B=64 x T=800, L=101, V=63"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_tle_lm: needs a CUDA device (no CPU measurement)")
    pkg = __import__("__graft_entry__").load_package()
    dev = torch.device("cuda", 0)
    V = ICLR["num_phonemes"]
    S, start, arcs = LO.char_ngram(V, seed=7, n_tri=60, dup=6, dead=2)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "lm.fst")
        cmap = LO.to_file(path, V, S, start, arcs, seed=2)
        lm = dict(path=path, weight=0.15)
        recs = {}
        for c in CRITERIA:
            recs[c] = make(pkg, dev, c, None, None)
            recs[c + "+lm"] = make(pkg, dev, c, lm, cmap)
    rng = np.random.RandomState(99)
    T = 300
    lens = rng.randint(int(0.6 * T), T + 1, size=8)
    lens[0] = T
    inputs = [{"recordings": rng.normal(size=(int(t), ICLR["num_features"])).astype(np.float32)} for t in lens]
    out = {"gpu": bench.gpu_identity(0),
           "model": "iclr_reward shape: 123 features, 3 x BiGRU(256), subsample [1,1,1], V=63, Maxout(2)",
           "lm": {"states": S, "arcs": sum(len(a) for a in arcs), "weight": 0.15, "no_transition_cost": 1e12},
           "search_workload": "8 utterances x <= %d frames, max_decoded_length_scale %g" % (T, SCALE)}
    for beam in (10, 200):
        out["search_beam%d" % beam] = time_search(torch, dev, recs, inputs, beam, args.steps, args.warmup)
    out["cost_matrix"] = time_cost(torch, dev, recs, max(args.steps, 5), args.warmup)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
