"""Cost of dropout and weight noise (regularization.dropout / noise): training steps with each on, alternating in one
process, on the GPU.

    python tools/bench_regularization.py [--steps 9] [--warmup 2]

One recognizer and five GradientDescents, each with its own setting (momentum + AdaDelta + StepClipping): no
regularisation, dropout, weight noise (level 0.075, the WSJ recipes' value), the alignment penalty (coefficient 1) and
all three (GradientDescent drops dropout beside noise, as the reference does, so "all" runs noise and the penalty).  process_batch is timed with
CUDA events and a synchronisation per step, the variants alternating step by step, on bench.py --mode train's step
(B=64 x T=1500, WSJ architecture, L=190).  Then the "dropout", "weight_noise" and "penalty" kernel classes per step, from a
profiled pass of their own.  One JSON object with the card's name and power limit.  Writes nothing.
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools.bench_adaptive_noise import make  # noqa: E402

VARIANTS = [("off", None), ("dropout", dict(dropout=True)), ("noise", dict(noise=0.075)),
            ("penalty", dict(penalty_coof=1.0)), ("all", dict(noise=0.075, penalty_coof=1.0))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_regularization: needs a CUDA device")
    import __graft_entry__ as graft
    pkg = graft.load_package()
    lib = pkg._lib.load()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    net, W = dict(bench.NET, attention_type="content_and_conv"), dict(bench.TRAIN_WORKLOAD)
    chain = dict(gradient_threshold=100.0, rules=["momentum", "adadelta"], scale=1.0, momentum=0.0, decay_rate=0.95,
                 epsilon=1e-8)
    # one recognizer: five training arenas of this size would not fit the card together.  Switching a variant
    # (initialize: optimizer state, regularisation buffers) happens outside the timed window.
    rec = make(pkg, dev, net)
    algos = {name: pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(chain), regularization=reg)
             for name, reg in VARIANTS}
    x, m, labels, lm = bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"], seed=11)
    batch = dict(recordings=x, recordings_mask=m, labels=labels, labels_mask=lm)

    def step(a):
        a.initialize()
        # a weight-noise update leaves the weights packed from its noisy copy: pack the means here, outside the timed
        # window, so that no variant pays for the one before it
        pkg._lib.check(lib.lvsr_model_finalize(rec._require_ready()))
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        a.process_batch(batch)
        e1.record()
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1)

    for _ in range(args.warmup):
        for a in algos.values():
            step(a)
    ms = {k: [] for k in algos}
    for _ in range(args.steps):
        for k, a in algos.items():
            ms[k].append(step(a))
    med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
    out = {"gpu": bench.gpu_identity(0), "workload": W}
    for k in algos:
        out["ms_per_step_" + k] = round(med[k], 3)
        out["ms_per_step_%s_min" % k] = round(min(ms[k]), 3)
        if k != "off":
            out["overhead_pct_" + k] = round(100.0 * (med[k] / med["off"] - 1.0), 2)
    # the kernel classes in a pass of their own (event timing slows the host)
    tot, cnt = C.c_double(), C.c_int64()
    classes = (b"dropout", b"weight_noise", b"penalty")
    for cls in classes:
        lib.lvsr_profile_read(cls, C.byref(tot), C.byref(cnt))
    lib.lvsr_profile_enable(1)
    for name in ("dropout", "all"):
        algos[name].initialize()
        for _ in range(args.steps):
            algos[name].process_batch(batch)
    torch.cuda.synchronize(dev)
    lib.lvsr_profile_enable(0)
    for cls in classes:
        lib.lvsr_profile_read(cls, C.byref(tot), C.byref(cnt))
        out["%s_class_ms_per_step" % cls.decode()] = round(tot.value / args.steps, 4)
        out["%s_launches_per_step" % cls.decode()] = cnt.value / args.steps
    out["task_cost"] = {k: float(a.last_cost.item()) for k, a in algos.items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
