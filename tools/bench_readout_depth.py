"""Time the readout's post-merge depth on the GPU: the benchmarked model (bench.py's NET) with its Maxout(2) depth-1
readout against Rectifier readouts of post_merge_dims [256, 256] and [256, 256, 256], at bench.py's metric shape
(teacher-forced cost of B=64 x T=1000 frames), its training step at that shape and a beam search (beam 10) over
utterances of 800 frames.  Per shape: the call time from device events (median of --steps after --warmup), and the
per-class device time of the readout (lvsr_profile: "readout", the body "readout_body" and its backward
"readout_body_bwd") from a separate profiled run.  Prints one JSON line per (readout, shape) with the GPU's name and
power limit.

    python tools/bench_readout_depth.py [--steps 5] [--warmup 2] [--out readout_depth.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
import __graft_entry__ as graft  # noqa: E402

READOUTS = {"depth1_maxout2": ([256], "maxout"), "relu_256x2": ([256, 256], "relu"),
            "relu_256x3": ([256, 256, 256], "relu")}
CLASSES = ("readout", "readout_body", "readout_body_bwd")


def gpu_identity():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def make(pkg, dims, act, seed=1):
    net = dict(bench.NET)
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": net["num_features"]}, input_num_chars={}, eos_label=net["num_phonemes"] - 1,
        num_phonemes=net["num_phonemes"], dim_dec=net["dim_dec"], dims_bidir=net["dims_bidir"],
        subsample=net["subsample"], dim_matcher=net["dim_matcher"], conv_n=net["conv_n"],
        conv_num_filters=net["conv_num_filters"], post_merge_dims=dims,
        post_merge_activation=pkg.Maxout(2) if act == "maxout" else pkg.Rectifier(),
        enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent)
    rec.set_parameter_values(bench.init_values(rec.parameter_shapes(), seed=seed))
    return rec


def timed(torch, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def profiled(lib, torch, fn):
    lib.lvsr_profile_enable(1)
    fn()
    torch.cuda.synchronize()
    lib.lvsr_profile_enable(0)
    out = {}
    for cls in CLASSES:
        ms, n = ctypes.c_double(), ctypes.c_int64()
        lib.lvsr_profile_read(cls.encode(), ctypes.byref(ms), ctypes.byref(n))
        out[cls] = dict(ms=round(ms.value, 4), launches=int(n.value))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_readout_depth needs a GPU"
    pkg = graft.load_package()
    lib = pkg._lib.load()
    gpu = gpu_identity()
    W = bench.WORKLOAD
    x, m, labels, lm = bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"], seed=1234)
    rng = np.random.RandomState(5)
    utts = [rng.normal(size=(800, W["F"])).astype(np.float32) for _ in range(8)]
    lines = []
    for name, (dims, act) in READOUTS.items():
        rec = make(pkg, dims, act)
        algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
        batch = dict(zip(algo.SOURCES, (x, m, labels, lm)))
        rec.init_beam_search(10)
        shapes = {"metric_cost": lambda: rec.cost(x, m, labels, lm),
                  "train_step": lambda: algo.cost_and_gradients(batch),
                  "search_beam10_8x800": lambda: rec.beam_search_many([{"recordings": u} for u in utts],
                                                                    raise_on_failure=False)}
        for shape, fn in shapes.items():
            line = dict(readout=name, post_merge_dims=dims, activation=act, shape=shape,
                        ms=round(timed(torch, fn, args.steps, args.warmup), 3), classes=profiled(lib, torch, fn), gpu=gpu)
            print(json.dumps(line), flush=True)
            lines.append(line)
        del rec, algo
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
