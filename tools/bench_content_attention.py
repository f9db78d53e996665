"""Content-only attention against content_and_conv attention, on the GPU, alternating the two models in one process.

    python tools/bench_content_attention.py [--steps 10] [--warmup 3]

Prints one JSON line:
  * metric: lvsr_cost_matrix at the metric shape (B=64 x T=1000, WSJ encoder, M=512, L=125): persistent-decoder
    milliseconds per step (the "dec_scan" kernel class) and cost_matrix frames/s, for both attention types;
  * timit: the same at the TIMIT baseline shape (3 x BiGRU(256), no subsampling, V=63, B=16 x T=2000, L=60);
  * train: one lvsr_train_cost_and_grads call at configs[3] (B=64 x T=1500, WSJ architecture, L=190);
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

TIMIT = dict(num_features=40, dims_bidir=[256, 256, 256], subsample=[1, 1, 1], dim_dec=256, dim_matcher=256,
             conv_n=100, conv_num_filters=10, num_phonemes=63, post_merge_dims=[256], maxout_pieces=2)


def make(pkg, dev, net, attention_type):
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": net["num_features"]}, input_num_chars={}, eos_label=net["num_phonemes"] - 1,
        num_phonemes=net["num_phonemes"], dim_dec=net["dim_dec"], dims_bidir=net["dims_bidir"],
        subsample=net["subsample"], conv_n=net["conv_n"], conv_num_filters=net["conv_num_filters"],
        dim_matcher=net["dim_matcher"], post_merge_dims=net["post_merge_dims"], post_merge_activation=pkg.Maxout(2),
        attention_type=attention_type, enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent, device=dev)
    rec.set_parameter_values(bench.init_values(rec.parameter_shapes()))
    return rec


def prof_ms(lib, cls):
    tot, cnt = C.c_double(), C.c_int64()
    lib.lvsr_profile_read(cls.encode(), C.byref(tot), C.byref(cnt))
    return tot.value


def time_cost_matrix(torch, lib, recs, W, steps, warmup, seed):
    """cost_matrix of each model on the same encoded batch, the models alternating call by call."""
    x, m, labels, lm = bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"], seed=seed)
    dev = recs["content"].device
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
    # the persistent decoder alone (per-class CUDA events, in calls of their own)
    dec = {k: 0.0 for k in recs}
    for _ in range(steps):
        for k, r in recs.items():
            lib.lvsr_profile_enable(1)
            r.cost_matrix(y, ym, *enc[k])
            torch.cuda.synchronize(dev)
            lib.lvsr_profile_enable(0)
            dec[k] += prof_ms(lib, "dec_scan")
            for cls in ("gemm", "attention", "window", "dense", "readout"):
                prof_ms(lib, cls)
    out = {}
    for k in recs:
        med = sorted(ms[k])[len(ms[k]) // 2]
        out[k] = {"cost_matrix_ms_median": round(med, 3), "cost_matrix_ms_min": round(min(ms[k]), 3),
                  "decoder_us_per_step": round(dec[k] / steps / W["L"] * 1e3, 2),
                  "frames_per_s": round(W["B"] * W["T"] / (med * 1e-3))}
        out[k]["launch_status"] = recs[k].launch_status()
    return out


def time_train(torch, lib, recs, W, steps, warmup, seed):
    x, m, labels, lm = bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"], seed=seed)
    dev = recs["content"].device
    xd, md, yd, ymd = (torch.as_tensor(a, device=dev) for a in (x, m, labels, lm))
    out = {}
    bufs = {k: (torch.zeros(int(lib.lvsr_model_flat_size(r._require_ready())), device=dev),
                torch.zeros(1, device=dev)) for k, r in recs.items()}

    def step(k):
        r = recs[k]
        g, c = bufs[k]
        rc = lib.lvsr_train_cost_and_grads(r._require_ready(), xd.data_ptr(), md.data_ptr(), yd.data_ptr(), ymd.data_ptr(),
                                           W["T"], W["B"], W["L"], 1.0 / W["B"], c.data_ptr(), g.data_ptr(), r._stream())
        if rc != 0:
            raise RuntimeError(lib.lvsr_last_error().decode())
    for _ in range(warmup):
        for k in recs:
            step(k)
    torch.cuda.synchronize(dev)
    ms = {k: [] for k in recs}
    for _ in range(steps):
        for k in recs:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step(k)
            b.record()
            torch.cuda.synchronize(dev)
            ms[k].append(a.elapsed_time(b))
    for k in recs:
        med = sorted(ms[k])[len(ms[k]) // 2]
        out[k] = {"cost_and_grads_ms_median": round(med, 2), "cost_and_grads_ms_min": round(min(ms[k]), 2),
                  "frames_per_s": round(W["B"] * W["T"] / (med * 1e-3)), "cost": float(bufs[k][1].item())}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-train", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_content_attention: needs a CUDA device (no CPU measurement)")
    pkg = __import__("__graft_entry__").load_package()
    lib = pkg._lib.load()
    dev = torch.device("cuda", 0)
    result = {"gpu": bench.gpu_identity(0)}
    types = ("content", "content_and_conv")
    recs = {t: make(pkg, dev, bench.NET, t) for t in types}
    result["metric"] = dict(time_cost_matrix(torch, lib, recs, bench.WORKLOAD, args.steps, args.warmup, 1234),
                            shape="B=64 x T=1000, WSJ encoder, M=512, L=125")
    if not args.skip_train:
        result["train"] = dict(time_train(torch, lib, recs, bench.TRAIN_WORKLOAD, max(3, args.steps // 2), 2, 4321),
                               shape="configs[3]: B=64 x T=1500, WSJ architecture, L=190")
    del recs
    recs = {t: make(pkg, dev, TIMIT, t) for t in types}
    W = dict(B=16, T=2000, F=40, L=60, V=63)
    result["timit"] = dict(time_cost_matrix(torch, lib, recs, W, args.steps, args.warmup, 777),
                           shape="3 x BiGRU(256), subsample [1,1,1], V=63, B=16 x T=2000, M=256, L=60")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
