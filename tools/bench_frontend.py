"""The filterbank front end at the metric shape, beside the encoder forward of bench.py's network on its output.

    python tools/bench_frontend.py [--steps 20] [--warmup 3]

64 utterances x 160 240 samples at 16 kHz (1000 frames each), already on the device as float32 in int16 units, go
through Fbank.compute for the recipes' fbank_dd (40 bins + energy, deltas of order 2: 123 features, with global
CMVN) and for bench.py's 40-feature input (40 bins, no energy, no deltas).  Per configuration one JSON field:
  * us_median / us_min: the whole compute call (CUDA events, L2 flushed before each call);
  * kernel_us: the two front-end kernels alone, one profiled call (lvsr_profile_read "fbank");
  * bytes: the samples read plus the features and mask written, the least traffic the computation needs; GBps: those
    bytes over the median call, and their share of the H100 SXM data sheet's 3.35 TB/s of HBM3;
  * encoder_us: rec.encode of bench.NET (4 x 256 BiGRU, subsampling [1, 1, 2, 2]) on the features, and ratio: front
    end over encoder.
  * gpu: the card's name, power limit and maximum SM clock, which every number depends on.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

B, N = 64, 160240
HBM_BPS = 3.35e12


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
    return ms[len(ms) // 2] * 1e3, ms[0] * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_frontend: needs a CUDA device (no CPU measurement)")
    pkg = __import__("__graft_entry__").load_package()
    lib = pkg._lib.load()
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    rng = np.random.RandomState(1234)
    t = np.arange(N) / 16000.0
    waves = (rng.normal(0, 600, size=(B, N)) + 3000 * np.sin(2 * np.pi * rng.uniform(200, 3000, size=(B, 1)) * t))
    x = torch.as_tensor(np.clip(np.round(waves), -32768, 32767).astype(np.float32), device=dev)
    out = {"gpu": bench.gpu_identity(0), "shape": "B=%d x N=%d samples (T=1000)" % (B, N)}
    configs = {"fbank_dd_123": pkg.FbankOptions(), "fbank_40": pkg.FbankOptions(use_energy=False, delta_order=0)}
    tot, cnt = C.c_double(), C.c_int64()
    for name, opts in configs.items():
        fb = pkg.Fbank(opts, dev)
        feats, mask = fb.compute(x)
        cmvn = pkg.GlobalCmvn(fb)
        cmvn.accumulate(feats, mask)
        T, D = feats.shape[0], feats.shape[2]
        us_med, us_min = timed(torch, dev, flush, lambda: fb.compute(x, cmvn=cmvn), args.warmup, args.steps)
        lib.lvsr_profile_read(b"fbank", C.byref(tot), C.byref(cnt))
        lib.lvsr_profile_enable(1)
        fb.compute(x, cmvn=cmvn)
        torch.cuda.synchronize(dev)
        lib.lvsr_profile_enable(0)
        lib.lvsr_profile_read(b"fbank", C.byref(tot), C.byref(cnt))
        nbytes = B * N * 4 + T * B * D * 4 + T * B * 4
        feats, mask = fb.compute(x, cmvn=cmvn)
        net = dict(bench.NET)
        rec = pkg.SpeechRecognizer(
            input_dims={"recordings": D}, input_num_chars={}, eos_label=31, num_phonemes=32, dim_dec=net["dim_dec"],
            dims_bidir=net["dims_bidir"], subsample=net["subsample"], conv_n=net["conv_n"],
            conv_num_filters=net["conv_num_filters"], dim_matcher=net["dim_matcher"],
            post_merge_dims=net["post_merge_dims"], post_merge_activation=pkg.Maxout(2),
            enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent, device=dev)
        rec.set_parameter_values(bench.init_values(rec.parameter_shapes()))
        enc_med, _ = timed(torch, dev, flush, lambda: rec.encode(feats, mask), 2, max(3, args.steps // 4))
        out[name] = dict(T=T, D=D, us_median=round(us_med, 1), us_min=round(us_min, 1),
                         kernel_us=round(tot.value * 1e3, 1), bytes=nbytes, GBps=round(nbytes / us_med / 1e3, 1),
                         hbm_share=round(nbytes / (us_med * 1e-6) / HBM_BPS, 3), encoder_us=round(enc_med, 1),
                         ratio=round(us_med / enc_med, 4))
        del rec, fb, cmvn
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
