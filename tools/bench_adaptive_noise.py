"""Cost of adaptive weight noise: training steps with and without it, alternating in one process, on the GPU.

    python tools/bench_adaptive_noise.py [--steps 8] [--warmup 2]

Two recognizers with the same parameters, one GradientDescent each (momentum + AdaDelta + StepClipping, the TIMIT
recipe's chain); process_batch is timed with CUDA events and a synchronisation per step, the two alternating step by
step.  Workloads:
  * configs3: bench.py's training step (B=64 x T=1500, WSJ architecture, L=190);
  * timit_b8 / timit_b1: 3 x BiGRU(256), 123 features, content attention, V=63, T=400, L=50, batch 8 and batch 1
    (batch 1 is the recipe's `main` stage).
Per workload one JSON object: ms per step with and without the noise (median), the overhead, the "noise" kernel class
per step (sample pass + prior reduction + gradient transform, from a profiled pass of its own), the bytes those
kernels must move (sample: read p, ls2, write p_noisy; transform: read g, p, ls2, write both gradients = 32 B per
parameter) over that time against the H100 SXM's 3.35 TB/s, and the card's name and power limit.  Writes nothing.
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

TIMIT = dict(num_features=123, dims_bidir=[256, 256, 256], subsample=[1, 1, 1], dim_dec=256, dim_matcher=256,
             conv_n=100, conv_num_filters=10, num_phonemes=63, post_merge_dims=[256], maxout_pieces=2,
             attention_type="content")
WORKLOADS = [("configs3", dict(bench.NET, attention_type="content_and_conv"), dict(bench.TRAIN_WORKLOAD)),
             ("timit_b8", TIMIT, dict(B=8, T=400, F=123, L=50, V=63)),
             ("timit_b1", TIMIT, dict(B=1, T=400, F=123, L=50, V=63))]
HBM_BYTES_PER_S = 3.35e12


def make(pkg, dev, net):
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": net["num_features"]}, input_num_chars={}, eos_label=net["num_phonemes"] - 1,
        num_phonemes=net["num_phonemes"], dim_dec=net["dim_dec"], dims_bidir=net["dims_bidir"],
        subsample=net["subsample"], conv_n=net["conv_n"], conv_num_filters=net["conv_num_filters"],
        dim_matcher=net["dim_matcher"], post_merge_dims=net["post_merge_dims"], post_merge_activation=pkg.Maxout(2),
        attention_type=net["attention_type"], enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent,
        device=dev)
    rec.set_parameter_values(bench.init_values(rec.parameter_shapes()))
    return rec


def run(pkg, torch, lib, dev, net, W, steps, warmup):
    chain = dict(gradient_threshold=100.0, rules=["momentum", "adadelta"], scale=1.0, momentum=0.0, decay_rate=0.95,
                 epsilon=1e-8)
    algos = {}
    for k in ("plain", "noise"):
        an = dict(num_examples=3696, init_sigma=1e-6, model_cost_coefficient=0.1) if k == "noise" else None
        algos[k] = pkg.GradientDescent(recognizer=make(pkg, dev, net), step_rule=pkg.step_rule_from_config(chain),
                                       adaptive_noise=an)
        algos[k].initialize()
    x, m, labels, lm = bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"], seed=11)
    batch = dict(recordings=x, recordings_mask=m, labels=labels, labels_mask=lm)
    for _ in range(warmup):
        for a in algos.values():
            a.process_batch(batch)
    torch.cuda.synchronize(dev)
    ms = {k: [] for k in algos}
    for _ in range(steps):
        for k, a in algos.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            a.process_batch(batch)
            e1.record()
            torch.cuda.synchronize(dev)
            ms[k].append(e0.elapsed_time(e1))
    # the "noise" class in a pass of its own (event timing slows the host)
    tot, cnt = C.c_double(), C.c_int64()
    lib.lvsr_profile_read(b"noise", C.byref(tot), C.byref(cnt))
    lib.lvsr_profile_enable(1)
    for _ in range(steps):
        algos["noise"].process_batch(batch)
    torch.cuda.synchronize(dev)
    lib.lvsr_profile_enable(0)
    lib.lvsr_profile_read(b"noise", C.byref(tot), C.byref(cnt))
    noise_ms = tot.value / steps
    n = sum(int(c) for _, c in algos["noise"]._offsets().values())
    med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
    moved = 32.0 * n
    return {"parameters": n, "ms_per_step_plain": round(med["plain"], 3), "ms_per_step_noise": round(med["noise"], 3),
            "ms_per_step_plain_min": round(min(ms["plain"]), 3), "ms_per_step_noise_min": round(min(ms["noise"]), 3),
            "overhead_pct": round(100.0 * (med["noise"] / med["plain"] - 1.0), 2),
            "noise_class_ms_per_step": round(noise_ms, 4), "noise_launches_per_step": cnt.value / steps,
            "noise_bytes_per_step": int(moved),
            "noise_bytes_per_s": round(moved / (noise_ms * 1e-3)) if noise_ms > 0 else None,
            "noise_share_of_3.35TBps": round(moved / (noise_ms * 1e-3) / HBM_BYTES_PER_S, 3) if noise_ms > 0 else None,
            "task_cost_noise": float(algos["noise"].last_cost.item()), "noise_stats": algos["noise"].noise_stats()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", default=None, help="comma-separated workload names")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_adaptive_noise: needs a CUDA device")
    import __graft_entry__ as graft
    pkg = graft.load_package()
    lib = pkg._lib.load()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    out = {"gpu": bench.gpu_identity(0)}
    for name, net, W in WORKLOADS:
        if args.only and name not in args.only.split(","):
            continue
        out[name] = run(pkg, torch, lib, dev, net, W, args.steps, args.warmup)
        out[name]["workload"] = W
    print(json.dumps(out))


if __name__ == "__main__":
    main()
