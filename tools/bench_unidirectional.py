"""A forward-only encoder (net.bidir: False) against the bidirectional one of the same widths, on the GPU.

    python tools/bench_unidirectional.py [--steps 10] [--warmup 2] [--train-steps 5]

Both models take bench.NET (4 x 256, subsampling [1, 1, 2, 2]) with bench.py's initial values; the forward-only one
has half the encoder's scan clusters and projection columns and an encoded width of 256 instead of 512.  Prints one
JSON line:
  * forward: the encoder + teacher-forced cost (as bench.py's metric mode runs them:
    encode, then cost_matrix) at B = 64 x T = 1000, and
  * train: the training step (GradientDescent.process_batch) at B = 64 x T = 1500,
  each as the median and minimum of reps that alternate between the two models (CUDA events, L2 flushed before each
  call), with per-class times of one profiled rep (lvsr_profile_read: "bigru", "gemm", "bigru_bwd", "gemm_tn") and
  the encoder plan of every layer (scan kernel, rows per cluster, clusters, waves);
  * gpu: the card's name, power limit and maximum SM clock, which every number depends on.
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

CLASSES = (b"bigru", b"gemm", b"bigru_bwd", b"gemm_tn")


def recognizer(pkg, dev, W, bidir):
    N = bench.NET
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": W["F"]}, input_num_chars={}, eos_label=W["V"] - 1, num_phonemes=W["V"],
        dim_dec=N["dim_dec"], dims_bidir=N["dims_bidir"], subsample=N["subsample"], conv_n=N["conv_n"],
        conv_num_filters=N["conv_num_filters"], dim_matcher=N["dim_matcher"], post_merge_dims=N["post_merge_dims"],
        post_merge_activation=pkg.Maxout(2), enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent,
        bidir=bidir, device=dev)
    rec.set_parameter_values(bench.init_values(rec.parameter_shapes()))
    return rec


def one(torch, dev, flush, fn):
    flush.fill_(1)
    torch.cuda.synchronize(dev)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize(dev)
    return a.elapsed_time(b)


def profiled(torch, dev, lib, fn):
    tot, cnt = C.c_double(), C.c_int64()
    for cls in CLASSES:
        lib.lvsr_profile_read(cls, C.byref(tot), C.byref(cnt))
    lib.lvsr_profile_enable(1)
    fn()
    torch.cuda.synchronize(dev)
    lib.lvsr_profile_enable(0)
    out = {}
    for cls in CLASSES:
        lib.lvsr_profile_read(cls, C.byref(tot), C.byref(cnt))
        out[cls.decode() + "_ms"] = round(tot.value, 3)
    return out


def compare(torch, dev, flush, lib, calls, plans, warmup, steps):
    """calls: {name: fn}; reps alternate between them."""
    for _ in range(warmup):
        for fn in calls.values():
            fn()
    ms = {k: [] for k in calls}
    for _ in range(steps):
        for k, fn in calls.items():
            ms[k].append(one(torch, dev, flush, fn))
    out = {}
    for k, v in ms.items():
        v.sort()
        out[k] = dict(ms_median=round(v[len(v) // 2], 3), ms_min=round(v[0], 3), profile=profiled(torch, dev, lib, calls[k]),
                      layers=plans[k]())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--train-steps", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_unidirectional: needs a CUDA device (no CPU measurement)")
    pkg = __import__("__graft_entry__").load_package()
    lib = pkg._lib.load()
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    out = {"gpu": bench.gpu_identity(0), "net": bench.NET["dims_bidir"]}

    def plan_of(rec):
        return lambda: [(p["bigru"], p["rb"], p["clusters"], p["waves"], p["proj"], p["overlap"])
                        for p in rec.encoder_plan()]

    W = bench.WORKLOAD
    x, m, labels, lm = bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"], seed=1234)
    xd, md = torch.as_tensor(x, device=dev), torch.as_tensor(m, device=dev)
    ld, lmd = torch.as_tensor(labels, device=dev), torch.as_tensor(lm, device=dev)
    recs = {"bidir": recognizer(pkg, dev, W, True), "unidir": recognizer(pkg, dev, W, False)}

    def forward(rec):
        def fn():
            att, attm = rec.encode(xd, md)
            rec.cost_matrix(ld, lmd, att, attm)
        return fn

    out["forward_shape"] = "B=%d x T=%d" % (W["B"], W["T"])
    out["forward"] = compare(torch, dev, flush, lib, {k: forward(r) for k, r in recs.items()},
                             {k: plan_of(r) for k, r in recs.items()}, args.warmup, args.steps)
    del recs
    torch.cuda.empty_cache()

    TW = bench.TRAIN_WORKLOAD
    x, m, labels, lm = bench.synthetic_batch(TW["B"], TW["T"], TW["F"], TW["L"], TW["V"], seed=4321)
    batch = dict(zip(("recordings", "recordings_mask", "labels", "labels_mask"),
                     (torch.as_tensor(a, device=dev) for a in (x, m, labels, lm))))
    recs, algos = {}, {}
    for name, bidir in (("bidir", True), ("unidir", False)):
        recs[name] = recognizer(pkg, dev, TW, bidir)
        algos[name] = pkg.GradientDescent(recognizer=recs[name],
                                          step_rule=pkg.step_rule_from_config(bench.TRAIN_CONF, dict(max_norm=1.0)))
        algos[name].initialize()
    out["train_shape"] = "B=%d x T=%d" % (TW["B"], TW["T"])
    out["train"] = compare(torch, dev, flush, lib, {k: (lambda a=a: a.process_batch(batch)) for k, a in algos.items()},
                           {k: plan_of(r) for k, r in recs.items()}, 1, args.train_steps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
