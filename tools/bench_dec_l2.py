"""The persistent decoder's L2 priority of P and H (LVSR_DEC_L2), on the GPU, the settings alternating call by call.

    python tools/bench_dec_l2.py [--calls 10] [--warmup 2] [--settings "off;auto;1,0.2;..."] [--no-trace]

Two workloads, each on one fixed encoded batch (bench.py's generators and seeds):
  * metric: lvsr_cost_matrix at the metric shape (B=64 x T=1000, WSJ encoder, M=E=512, T'=250, L=125);
  * taped: the training step's forward, lvsr_cost_matrix with weights, energies, states and weighted averages kept
    (configs[3]: B=64 x T=1500, T'=375, L=190).
Each setting (`off`: plain loads; `auto`: the planner's default; fP,fH: those shares of P's and H's lines keep the
normal L2 priority, the rest is evicted first; default: off, auto and fP in {0, .25, .5, .75, 1}
x fH in {0, .1, .2, .3}) runs once per round, the settings in turn, with the L2 flushed (256 MiB write) before every
call; CUDA events time each call and the median of --calls rounds is reported with decoder_plan()["l2_evict_first_kb"].
Unless --no-trace, the LVSR_DEC_TRACE per-phase split (µs per step) of one more call is recorded for off, auto and
1,0.  The card's name, power limit and maximum SM clock are printed with the numbers.  The library is the in-tree
build, or LVSR_B200_LIB's.  Prints one JSON line; nothing is written anywhere.
"""
import argparse
import json
import os
import re
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

GRID = ["off", "auto"] + ["%g,%g" % (fp, fh) for fp in (0, .25, .5, .75, 1) for fh in (0, .1, .2, .3)]


def set_l2(setting):
    if setting == "auto":
        os.environ.pop("LVSR_DEC_L2", None)
    else:
        os.environ["LVSR_DEC_L2"] = setting


def make(pkg, dev):
    net = bench.NET
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": net["num_features"]}, input_num_chars={}, eos_label=net["num_phonemes"] - 1,
        num_phonemes=net["num_phonemes"], dim_dec=net["dim_dec"], dims_bidir=net["dims_bidir"],
        subsample=net["subsample"], conv_n=net["conv_n"], conv_num_filters=net["conv_num_filters"],
        dim_matcher=net["dim_matcher"], post_merge_dims=net["post_merge_dims"], post_merge_activation=pkg.Maxout(2),
        enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent, device=dev)
    rec.set_parameter_values(bench.init_values(rec.parameter_shapes()))
    return rec


def traced(fn):
    """(fn's stderr, from the C library's fprintf) with stderr sent to a temporary file for the call"""
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+b") as f:
        os.dup2(f.fileno(), 2)
        try:
            fn()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        return f.read().decode("utf-8", "replace")


def phase_split(text):
    """the LVSR_DEC_TRACE lines of CTA 0 and its attention row as {phase: µs per step}"""
    out = {}
    for line in text.splitlines():
        if "CTA first:" in line or "attention row 0:" in line:
            out.update({k: float(v) for k, v in re.findall(r"(\w+)=([0-9.]+)us", line)})
    return out


def run(torch, rec, W, seed, return_all, settings, calls, warmup, trace, flush):
    x, m, labels, lm = bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"], seed=seed)
    dev = rec.device
    y, ym = torch.as_tensor(labels, device=dev), torch.as_tensor(lm, device=dev)
    att, attm = rec.encode(x, m)

    def call():
        return rec.cost_matrix(y, ym, att, attm, return_all=return_all)
    ms = {s: [] for s in settings}
    plans = {}
    for r in range(warmup + calls):
        for s in settings:
            set_l2(s)
            flush.fill_(1)
            torch.cuda.synchronize(dev)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            call()
            b.record()
            torch.cuda.synchronize(dev)
            if r >= warmup:
                ms[s].append(a.elapsed_time(b))
            plans[s] = rec.decoder_plan()
    out = {"settings": {}}
    for s in settings:
        med = sorted(ms[s])[len(ms[s]) // 2]
        out["settings"][s] = {"ms_median": round(med, 3), "ms_min": round(min(ms[s]), 3),
                              "ms_max": round(max(ms[s]), 3), "l2_evict_first_kb": plans[s]["l2_evict_first_kb"],
                              "kernel": plans[s]["kernel"]}
    if trace:
        out["trace_us_per_step"] = {}
        for s in trace:
            set_l2(s)
            os.environ["LVSR_DEC_TRACE"] = "1"
            flush.fill_(1)
            torch.cuda.synchronize(dev)
            text = traced(lambda: (call(), torch.cuda.synchronize(dev)))
            os.environ.pop("LVSR_DEC_TRACE")
            out["trace_us_per_step"][s] = phase_split(text)
    set_l2("auto")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--settings", default=None, help="settings separated by semicolons (default: the sweep grid)")
    ap.add_argument("--no-trace", action="store_true")
    ap.add_argument("--skip-taped", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_dec_l2: needs a CUDA device (no CPU measurement)")
    settings = args.settings.split(";") if args.settings else GRID
    for s in settings:
        if s not in ("off", "auto") and not re.fullmatch(r"[0-9.]+,[0-9.]+", s):
            raise SystemExit("bench_dec_l2: setting %r: expected off, auto or fP,fH" % s)
    trace = None if args.no_trace else ["off", "auto", "1,0"]
    pkg = __import__("__graft_entry__").load_package()
    lib_path = pkg._lib.LIB_PATH
    dev = torch.device("cuda", 0)
    props = torch.cuda.get_device_properties(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    result = {"gpu": bench.gpu_identity(0), "l2_bytes": props.L2_cache_size, "library": os.path.basename(lib_path)}
    rec = make(pkg, dev)
    result["metric"] = dict(run(torch, rec, bench.WORKLOAD, 1234, False, settings, args.calls, args.warmup, trace,
                                flush), shape="B=64 x T=1000, T'=250, M=E=512, L=125")
    if not args.skip_taped:
        result["taped"] = dict(run(torch, rec, bench.TRAIN_WORKLOAD, 4321, True, settings, args.calls, args.warmup,
                                   trace, flush), shape="configs[3] forward with the tape: B=64 x T=1500, T'=375, L=190")
    os.environ.pop("LVSR_DEC_L2", None)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
