"""Cost of the bottom MLP: the forward cost and the training step with and without bottom.dims [256] (Rectifier),
alternating in one process, on the GPU.

    python tools/bench_bottom.py [--steps 8] [--warmup 2]

Two recognizers of bench.py's WSJ architecture with the same encoder and decoder parameters, one of them with the
bottom MLP in front of the encoder (so its encoder layer 0 takes 256 features instead of 40).  Timed with CUDA events
and a synchronisation per call, the two alternating call by call:
  * forward: encode + cost_matrix on device buffers at bench.py's metric shape (B=64 x T=1000);
  * train: GradientDescent.process_batch at bench.py --mode train's shape (B=64 x T=1500, L=190).
Then a profiled pass of the model with the bottom gives the "bottom" (its forward GEMM + activation) and "bottom_bwd"
(its backward) kernel classes per call.  The difference of the two models' times also holds encoder layer 0's wider
projection (K = 256 instead of 40) and its input gradient, which only a bottom needs.  One JSON line, with the card's
name and power limit.  Writes nothing.
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

BOTTOM = dict(dims=[256])


def make(pkg, dev, W, bottom):
    net = bench.NET
    kw = dict(bottom=dict(BOTTOM, activation=pkg.Rectifier())) if bottom else {}
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": W["F"]}, input_num_chars={}, eos_label=W["V"] - 1, num_phonemes=W["V"],
        dim_dec=net["dim_dec"], dims_bidir=net["dims_bidir"], subsample=net["subsample"], conv_n=net["conv_n"],
        conv_num_filters=net["conv_num_filters"], dim_matcher=net["dim_matcher"], post_merge_dims=net["post_merge_dims"],
        post_merge_activation=pkg.Maxout(2), enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent,
        device=dev, **kw)
    rec.set_parameter_values(bench.init_values(rec.parameter_shapes()))
    return rec


def timed(torch, dev, fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize(dev)
    return e0.elapsed_time(e1)


def profiled(torch, dev, lib, fn, steps):
    tot, cnt = C.c_double(), C.c_int64()
    for cls in (b"bottom", b"bottom_bwd"):
        lib.lvsr_profile_read(cls, C.byref(tot), C.byref(cnt))
    lib.lvsr_profile_enable(1)
    for _ in range(steps):
        fn()
    torch.cuda.synchronize(dev)
    lib.lvsr_profile_enable(0)
    out = {}
    for cls in (b"bottom", b"bottom_bwd"):
        lib.lvsr_profile_read(cls, C.byref(tot), C.byref(cnt))
        out[cls.decode() + "_ms_per_call"] = round(tot.value / steps, 4)
    return out


def compare(torch, dev, lib, calls, steps, warmup):
    for _ in range(warmup):
        for fn in calls.values():
            fn()
    torch.cuda.synchronize(dev)
    ms = {k: [] for k in calls}
    for _ in range(steps):
        for k, fn in calls.items():
            ms[k].append(timed(torch, dev, fn))
    med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
    out = {"ms_plain": round(med["plain"], 3), "ms_bottom": round(med["bottom"], 3),
           "ms_plain_min": round(min(ms["plain"]), 3), "ms_bottom_min": round(min(ms["bottom"]), 3),
           "added_ms": round(med["bottom"] - med["plain"], 3),
           "added_pct": round(100.0 * (med["bottom"] / med["plain"] - 1.0), 2)}
    out.update(profiled(torch, dev, lib, calls["bottom"], steps))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_bottom: needs a CUDA device")
    import __graft_entry__ as graft
    pkg = graft.load_package()
    lib = pkg._lib.load()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    out = {"gpu": bench.gpu_identity(0), "bottom": dict(BOTTOM, activation="Rectifier")}

    W = dict(bench.WORKLOAD)
    recs = {k: make(pkg, dev, W, k == "bottom") for k in ("plain", "bottom")}
    x, m, labels, lm = (torch.as_tensor(a, device=dev) for a in
                        bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"], seed=11))

    def forward(rec):
        def fn():
            att, attm = rec.encode(x, m)
            rec.cost_matrix(labels, lm, att, attm)
        return fn
    out["forward"] = compare(torch, dev, lib, {k: forward(r) for k, r in recs.items()}, args.steps, args.warmup)
    out["forward"]["workload"] = W
    del recs

    W = dict(bench.TRAIN_WORKLOAD)
    algos = {}
    for k in ("plain", "bottom"):
        algos[k] = pkg.GradientDescent(recognizer=make(pkg, dev, W, k == "bottom"),
                                       step_rule=pkg.step_rule_from_config(bench.TRAIN_CONF, dict(max_norm=1.0)))
        algos[k].initialize()
    names = ("recordings", "recordings_mask", "labels", "labels_mask")
    batch = dict(zip(names, (torch.as_tensor(a, device=dev) for a in
                             bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"], seed=4321))))
    out["train"] = compare(torch, dev, lib, {k: (lambda a=a: a.process_batch(batch)) for k, a in algos.items()},
                           args.steps, args.warmup)
    out["train"]["workload"] = W
    print(json.dumps(out))


if __name__ == "__main__":
    main()
