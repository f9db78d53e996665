"""The encoder forward with each projection streamed beside the previous layer's BiGRU scan against the projection
after the scan (LVSR_ENC_OVERLAP=0), on the GPU, alternating the two call by call in one process.

    python tools/bench_encoder_overlap.py [--steps 20] [--warmup 3] [--batch 64] [--frames 1000] [--trace DIR]

Prints one JSON line, per mode ("overlap", "serial"):
  * encode_ms_median / encode_ms_min: lvsr_encoder_forward alone (CUDA events, L2 flushed before each call);
  * kernel_ms: the per-class CUDA-event times of a profiled call ("bigru" covers a scan and the projection tiles done
    beside it, "gemm" the projections and the tiles done after the scans);
  * kernels_us: torch.profiler durations of one call, summed per kernel name -- bigru_mma_kernel alone shows whether
    the concurrent GEMM's traffic slows the scans; overlap_us: how long gemm_f16_stream_kernel ran while a scan ran;
  * plan: per layer (overlap, tiles done beside the scan, tiles done after it).
The workload is bench.py's metric encoder (WSJ architecture, B=64 x T=1000 by default) on its synthetic inputs;
--trace DIR also writes the chrome trace of the profiled call with the overlap on.  `gpu` names the card, its power
limit and maximum SM clock, which every number depends on.
"""
import argparse
import ctypes as C
import json
import os
import re
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

MODES = {"overlap": None, "serial": "0"}   # value of LVSR_ENC_OVERLAP


def set_mode(mode):
    if MODES[mode] is None:
        os.environ.pop("LVSR_ENC_OVERLAP", None)
    else:
        os.environ["LVSR_ENC_OVERLAP"] = MODES[mode]


def kernel_trace(torch, rec, xd, md, path):
    """one encode under torch.profiler: {kernel name: summed us}, and the us gemm_f16_stream_kernel ran beside a scan"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rec.encode(xd, md)
        torch.cuda.synchronize()
    prof.export_chrome_trace(path)
    with open(path) as f:
        events = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
    sums = {}
    for e in events:
        found = re.search(r"\w+_kernel\b", e["name"])
        name = found.group(0) if found else e["name"][:40]
        sums[name] = sums.get(name, 0.0) + e["dur"]
    scans = [(e["ts"], e["ts"] + e["dur"]) for e in events if "bigru_mma_kernel" in e["name"]]
    beside = 0.0
    for e in events:
        if "gemm_f16_stream_kernel" in e["name"]:
            a, b = e["ts"], e["ts"] + e["dur"]
            beside += sum(max(0.0, min(b, s1) - max(a, s0)) for s0, s1 in scans)
    return {k: round(v, 1) for k, v in sorted(sums.items())}, round(beside, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=bench.WORKLOAD["B"])
    ap.add_argument("--frames", type=int, default=bench.WORKLOAD["T"])
    ap.add_argument("--trace", metavar="DIR", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_encoder_overlap: needs a CUDA device (no CPU measurement)")
    pkg = __import__("__graft_entry__").load_package()
    lib = pkg._lib.load()
    dev = torch.device("cuda", 0)
    W, N = bench.WORKLOAD, bench.NET
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": W["F"]}, input_num_chars={}, eos_label=W["V"] - 1, num_phonemes=W["V"],
        dim_dec=N["dim_dec"], dims_bidir=N["dims_bidir"], subsample=N["subsample"], conv_n=N["conv_n"],
        conv_num_filters=N["conv_num_filters"], dim_matcher=N["dim_matcher"], post_merge_dims=N["post_merge_dims"],
        post_merge_activation=pkg.Maxout(2), enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent,
        device=dev)
    rec.set_parameter_values(bench.init_values(rec.parameter_shapes()))
    x, m, _, _ = bench.synthetic_batch(args.batch, args.frames, W["F"], W["L"], W["V"], seed=1234)
    xd, md = torch.as_tensor(x, device=dev), torch.as_tensor(m, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    for _ in range(args.warmup):
        for mode in MODES:
            set_mode(mode)
            rec.encode(xd, md)
    torch.cuda.synchronize(dev)
    ms = {k: [] for k in MODES}
    for _ in range(args.steps):
        for mode in MODES:
            set_mode(mode)
            flush.fill_(1)
            torch.cuda.synchronize(dev)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            rec.encode(xd, md)
            b.record()
            torch.cuda.synchronize(dev)
            ms[mode].append(a.elapsed_time(b))

    out = {"gpu": bench.gpu_identity(0), "shape": "B=%d x T=%d, WSJ encoder" % (args.batch, args.frames)}
    tmp = tempfile.mkdtemp()
    for mode in MODES:
        set_mode(mode)
        lib.lvsr_profile_enable(1)
        rec.encode(xd, md)
        torch.cuda.synchronize(dev)
        lib.lvsr_profile_enable(0)
        kernel_ms = {}
        for cls in ("gemm", "bigru"):
            tot, cnt = C.c_double(), C.c_int64()
            lib.lvsr_profile_read(cls.encode(), C.byref(tot), C.byref(cnt))
            kernel_ms[cls] = round(tot.value, 3)
        plan = [(p["overlap"], p["tiles_beside"], p["tiles_after"]) for p in rec.encoder_plan()]
        path = os.path.join(args.trace if args.trace and mode == "overlap" else tmp, "encode_%s.json" % mode)
        if args.trace:
            os.makedirs(args.trace, exist_ok=True)
        kernels_us, beside_us = kernel_trace(torch, rec, xd, md, path)
        v = sorted(ms[mode])
        out[mode] = {"encode_ms_median": round(v[len(v) // 2], 3), "encode_ms_min": round(v[0], 3),
                     "kernel_ms": kernel_ms, "kernels_us": kernels_us, "overlap_us": beside_us, "plan": plan}
    set_mode("overlap")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
