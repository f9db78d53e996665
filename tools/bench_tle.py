"""Task loss estimation (criterion mse_gain) against log-likelihood, on the GPU, alternating the two models in one
process.

    python tools/bench_tle.py [--steps 10] [--warmup 3]

Prints one JSON line:
  * reward_kernel: lvsr_tle_matrices alone (the "tle_reward" kernel class, CUDA events per launch) at B=64 with
    groundtruth and prediction of 125 symbols, V=32, and at 300 symbols, V=63;
  * metric: lvsr_cost_matrix at bench.py's metric shape (B=64 x T=1000, WSJ encoder, L=125, V=32) for both criteria:
    milliseconds per call, and the task-loss kernels' share ("tle_reward" + "tle_loss" classes);
  * iclr_reward: the same at the TIMIT iclr_reward shape (3 x BiGRU(256), subsample [1, 1, 1], V=63, B=64 x T=800,
    L=101);
  * gpu: card name, power limit and maximum SM clock, which every number depends on.
Synthetic inputs and parameters from fixed seeds (bench.py's generators); nothing is written anywhere.
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

ICLR = dict(num_features=40, dims_bidir=[256, 256, 256], subsample=[1, 1, 1], dim_dec=256, dim_matcher=512,
            conv_n=100, conv_num_filters=10, num_phonemes=63, post_merge_dims=[256], maxout_pieces=2)


def make(pkg, dev, net, criterion):
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": net["num_features"]}, input_num_chars={}, eos_label=net["num_phonemes"] - 1,
        num_phonemes=net["num_phonemes"], dim_dec=net["dim_dec"], dims_bidir=net["dims_bidir"],
        subsample=net["subsample"], conv_n=net["conv_n"], conv_num_filters=net["conv_num_filters"],
        dim_matcher=net["dim_matcher"], post_merge_dims=net["post_merge_dims"], post_merge_activation=pkg.Maxout(2),
        criterion=dict(name=criterion, min_reward=-5.0), enc_transition=pkg.GatedRecurrent,
        dec_transition=pkg.GatedRecurrent, device=dev)
    rec.set_parameter_values(bench.init_values(rec.parameter_shapes()))
    return rec


def prof_ms(lib, cls):
    tot, cnt = C.c_double(), C.c_int64()
    lib.lvsr_profile_read(cls.encode(), C.byref(tot), C.byref(cnt))
    return tot.value


def time_reward_kernel(torch, pkg, lib, rec, B, L, steps, warmup, seed):
    import numpy as np
    V, eos = rec.net["num_phonemes"], rec.eos_label
    rng = np.random.RandomState(seed)
    g = rng.randint(0, V - 1, size=(L, B))
    g[-1] = eos
    y = rng.randint(0, V - 1, size=(L, B))
    dev = rec.device
    g, y = torch.as_tensor(g, device=dev), torch.as_tensor(y, device=dev)
    out = torch.empty((2, L, B, V), dtype=torch.float32, device=dev)
    h = rec._require_ready()

    def run():
        pkg._lib.check(lib.lvsr_tle_matrices(h, g.data_ptr(), L, y.data_ptr(), L, B, out[0].data_ptr(), out[1].data_ptr(),
                                             rec._stream()))
    for _ in range(warmup):
        run()
    total = 0.0
    for _ in range(steps):
        lib.lvsr_profile_enable(1)
        run()
        torch.cuda.synchronize(dev)
        lib.lvsr_profile_enable(0)
        total += prof_ms(lib, "tle_reward")
    return {"B": B, "L": L, "V": V, "kernel_us": round(total / steps * 1e3, 2)}


def time_cost_matrix(torch, lib, recs, W, steps, warmup, seed):
    """cost_matrix of each criterion on the same encoded batch, the models alternating call by call."""
    x, m, labels, lm = bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"], seed=seed)
    dev = recs["log_likelihood"].device
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
    tle_ms = {k: 0.0 for k in recs}
    for _ in range(steps):
        for k, r in recs.items():
            lib.lvsr_profile_enable(1)
            r.cost_matrix(y, ym, *enc[k])
            torch.cuda.synchronize(dev)
            lib.lvsr_profile_enable(0)
            tle_ms[k] += prof_ms(lib, "tle_reward") + prof_ms(lib, "tle_loss")
            for cls in ("gemm", "attention", "window", "dense", "readout", "dec_scan"):
                prof_ms(lib, cls)
    out = {}
    for k in recs:
        med = sorted(ms[k])[len(ms[k]) // 2]
        out[k] = {"cost_matrix_ms_median": round(med, 3), "cost_matrix_ms_min": round(min(ms[k]), 3),
                  "tle_kernels_ms": round(tle_ms[k] / steps, 4)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_tle: needs a CUDA device (no CPU measurement)")
    pkg = __import__("__graft_entry__").load_package()
    lib = pkg._lib.load()
    dev = torch.device("cuda", 0)
    result = {"gpu": bench.gpu_identity(0)}
    kinds = ("log_likelihood", "mse_gain")
    recs = {k: make(pkg, dev, bench.NET, k) for k in kinds}
    result["reward_kernel"] = [time_reward_kernel(torch, pkg, lib, recs["mse_gain"], 64, 125, args.steps, args.warmup, 1)]
    W = bench.WORKLOAD
    result["metric"] = dict(time_cost_matrix(torch, lib, recs, W, args.steps, args.warmup, 1234),
                            shape="B=64 x T=1000, WSJ encoder, M=512, L=125, V=32")
    del recs
    recs = {k: make(pkg, dev, ICLR, k) for k in kinds}
    result["reward_kernel"].append(time_reward_kernel(torch, pkg, lib, recs["mse_gain"], 64, 300, args.steps,
                                                      args.warmup, 2))
    W = dict(B=64, T=800, F=40, L=101, V=63)
    result["iclr_reward"] = dict(time_cost_matrix(torch, lib, recs, W, args.steps, args.warmup, 777),
                                 shape="3 x BiGRU(256), subsample [1,1,1], V=63, B=64 x T=800, M=512, L=101")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
