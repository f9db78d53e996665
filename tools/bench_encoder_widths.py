"""The encoder forward and the training step at the encoder widths beyond 128 / 256, on the GPU.

    python tools/bench_encoder_widths.py [--steps 10] [--warmup 2] [--train-steps 3]

Prints one JSON line:
  * encode: per width D (every layer of bench.py's metric encoder set to D, subsampling [1, 1, 2, 2]), the encoder
    forward at bench.py's metric shape (B = 64 x T = 1000): frames_per_s (B * T over the median call, CUDA events, L2
    flushed before each call), encode_ms_median / encode_ms_min and, per layer, (kernel, CTAs per cluster, clusters,
    resident clusters, waves) from encoder_plan().  "256_ffma" is 256 with the tensor-core scan turned off
    (LVSR_BIGRU_MMA=0);
  * train: per width 256, 320 and 512, the training step (GradientDescent.process_batch) at bench.py --mode train's
    shape (B = 64 x T = 1500), step_ms_median / step_ms_min, and per layer (forward kernel, CTAs per cluster, waves,
    backward CTAs per cluster, weight-gradient path);
  * gpu: the card's name, power limit and maximum SM clock, which every number depends on.
Widths are measured one after another in one process on bench.py's synthetic inputs and initial values.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

ENCODE = {"192": 192, "256": 256, "256_ffma": 256, "320": 320, "384": 384, "512": 512}
TRAIN = (256, 320, 512)


def recognizer(pkg, dev, D):
    W, N = bench.WORKLOAD, bench.NET
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": W["F"]}, input_num_chars={}, eos_label=W["V"] - 1, num_phonemes=W["V"],
        dim_dec=N["dim_dec"], dims_bidir=[D] * len(N["dims_bidir"]), subsample=N["subsample"], conv_n=N["conv_n"],
        conv_num_filters=N["conv_num_filters"], dim_matcher=N["dim_matcher"], post_merge_dims=N["post_merge_dims"],
        post_merge_activation=pkg.Maxout(2), enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent,
        device=dev)
    rec.set_parameter_values(bench.init_values(rec.parameter_shapes()))
    return rec


def timed(torch, dev, flush, fn, warmup, steps):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(steps):
        flush.fill_(1)
        torch.cuda.synchronize(dev)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize(dev)
        ms.append(a.elapsed_time(b))
    ms.sort()
    return ms[len(ms) // 2], ms[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--train-steps", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_encoder_widths: needs a CUDA device (no CPU measurement)")
    pkg = __import__("__graft_entry__").load_package()
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    out = {"gpu": bench.gpu_identity(0), "encode": {}, "train": {}}

    W = bench.WORKLOAD
    x, m, _, _ = bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"], seed=1234)
    xd, md = torch.as_tensor(x, device=dev), torch.as_tensor(m, device=dev)
    out["encode_shape"] = "B=%d x T=%d" % (W["B"], W["T"])
    for name, D in ENCODE.items():
        if name.endswith("_ffma"):
            os.environ["LVSR_BIGRU_MMA"] = "0"
        rec = recognizer(pkg, dev, D)
        med, lo = timed(torch, dev, flush, lambda: rec.encode(xd, md), args.warmup, args.steps)
        plan = [(p["bigru"], p["cs"], p["clusters"], p["resident"], p["waves"]) for p in rec.encoder_plan()]
        out["encode"][name] = {"frames_per_s": round(W["B"] * W["T"] / (med / 1e3)), "encode_ms_median": round(med, 3),
                               "encode_ms_min": round(lo, 3), "layers": plan}
        os.environ.pop("LVSR_BIGRU_MMA", None)
        del rec
        torch.cuda.empty_cache()

    TW = bench.TRAIN_WORKLOAD
    x, m, labels, lm = bench.synthetic_batch(TW["B"], TW["T"], TW["F"], TW["L"], TW["V"], seed=4321)
    batch = dict(zip(("recordings", "recordings_mask", "labels", "labels_mask"),
                     (torch.as_tensor(a, device=dev) for a in (x, m, labels, lm))))
    out["train_shape"] = "B=%d x T=%d" % (TW["B"], TW["T"])
    for D in TRAIN:
        rec = recognizer(pkg, dev, D)
        algo = pkg.GradientDescent(recognizer=rec,
                                   step_rule=pkg.step_rule_from_config(bench.TRAIN_CONF, dict(max_norm=1.0)))
        algo.initialize()
        med, lo = timed(torch, dev, flush, lambda: algo.process_batch(batch), args.warmup, args.train_steps)
        plan = [(p["bigru"], p["cs"], p["waves"], p["bwd_cs"], p["wgrad"]) for p in rec.encoder_plan()]
        out["train"][str(D)] = {"step_ms_median": round(med, 2), "step_ms_min": round(lo, 2), "layers": plan,
                                "cost": float(algo.last_cost.item())}
        del algo, rec
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
