"""Beam search with and without shallow fusion of an FST language model, on the GPU, alternating in one process.

    python tools/bench_lm_search.py [--steps 3] [--warmup 1]

The workload is bench.py's configs[2] search (32 utterances x <= 800 frames, WSJ architecture, beam 10).  The LM is
a seeded synthetic character 4-gram over the 32 symbols with every history present: 33,825 states and 1,116,224
arcs; each history state backs off over epsilon to the next shorter one, so every hypothesis holds at most 4 FST
states.  It is written as an OpenFST vector file to a temporary directory and loaded through SpeechRecognizer(lm=...).
Prints one JSON line: utterances/s of both searches, the relative cost of fusion, the LM kernels' time per launch
(per-class CUDA events, in runs of their own) and the card name and power limit.  Nothing is written to the tree.
"""
import argparse
import json
import os
import struct
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

V = 32


def four_gram(seed=5):
    """(num_states, arcs per state as (ilabel, nextstate, weight) arrays in FST labels 1..V, 0 = epsilon).  State ids:
    0 = empty history, then histories of length 1, 2 and 3."""
    rng = np.random.RandomState(seed)
    b1, b2, b3 = 1, 1 + V, 1 + V + V * V
    S = b3 + V ** 3
    x = np.arange(V)
    arcs = [None] * S
    w = lambda n: rng.uniform(0.5, 4.0, size=n).astype(np.float32)
    bo = lambda: np.float32(rng.uniform(0.1, 1.0))
    arcs[0] = (x + 1, b1 + x, w(V))
    for c in range(V):
        arcs[b1 + c] = (np.append(x + 1, 0), np.append(b2 + c * V + x, 0), np.append(w(V), bo()))
    for h in range(V * V):                    # (b, c) -> (b, c, x)
        arcs[b2 + h] = (np.append(x + 1, 0), np.append(b3 + h * V + x, b1 + h % V), np.append(w(V), bo()))
    for h in range(V ** 3):                   # (a, b, c) -> (b, c, x)
        arcs[b3 + h] = (np.append(x + 1, 0), np.append(b3 + (h % (V * V)) * V + x, b2 + h % (V * V)),
                        np.append(w(V), bo()))
    return S, arcs


def write_vector_fst(path, S, arcs):
    dt = np.dtype([("ilabel", "<i4"), ("olabel", "<i4"), ("weight", "<f4"), ("nextstate", "<i4")])
    s = lambda t: struct.pack("<i", len(t)) + t.encode()
    syms = [("<eps>", 0)] + [("c%d" % k, k + 1) for k in range(V)]
    parts = [struct.pack("<i", 2125659606), s("vector"), s("standard"),
             struct.pack("<iiQqqq", 2, 1, 0, 0, S, sum(len(a[0]) for a in arcs)),
             struct.pack("<i", 2125658996), s("chars"), struct.pack("<qq", V + 1, len(syms))]
    parts += [s(k) + struct.pack("<q", v) for k, v in syms]
    for lab, nxt, wt in arcs:
        a = np.zeros(len(lab), dtype=dt)
        a["ilabel"], a["olabel"], a["weight"], a["nextstate"] = lab, lab, wt, nxt
        parts.append(struct.pack("<fq", 0.0, len(a)) + a.tobytes())
    with open(path, "wb") as f:
        f.write(b"".join(parts))
    return {"c%d" % k: k for k in range(V)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import ctypes as C
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_lm_search: needs a CUDA device (no CPU measurement)")
    pkg = __import__("__graft_entry__").load_package()
    lib = pkg._lib.load()
    dev = torch.device("cuda", 0)
    case, net = bench.SEARCH_CASES["config3_beam10"], bench.NET
    with tempfile.TemporaryDirectory() as tmp:
        S, arcs = four_gram()
        path = os.path.join(tmp, "lm4.fst")
        cmap = write_vector_fst(path, S, arcs)
        recs = {}
        for name, lm in (("no_lm", None), ("lm", dict(path=path, weight=0.5, no_transition_cost=20.0))):
            rec = pkg.SpeechRecognizer(
                input_dims={"recordings": 40}, input_num_chars={}, eos_label=31, num_phonemes=V, dim_dec=net["dim_dec"],
                dims_bidir=net["dims_bidir"], subsample=net["subsample"], conv_n=net["conv_n"],
                conv_num_filters=net["conv_num_filters"], dim_matcher=net.get("dim_matcher"),
                post_merge_dims=net["post_merge_dims"], post_merge_activation=pkg.Maxout(2),
                max_decoded_length_scale=case["scale"], data_prepend_eos=False, enc_transition=pkg.GatedRecurrent,
                dec_transition=pkg.GatedRecurrent, device=dev, lm=lm, character_map=cmap if lm else None)
            rec.set_parameter_values(bench.search_values(rec.parameter_shapes()))
            rec.init_beam_search(case["beam"])
            recs[name] = rec
        num_arcs = int(recs["lm"]._lm_tables["offsets"][-1])
    rng = np.random.RandomState(99)
    lens = rng.randint(int(0.6 * case["T"]), case["T"] + 1, size=case["U"])
    lens[0] = case["T"]
    inputs = [{"recordings": rng.normal(size=(int(t), 40)).astype(np.float32)} for t in lens]
    res = {}
    for _ in range(args.warmup):
        for name, rec in recs.items():
            res[name] = rec.beam_search_many(inputs, raise_on_failure=False)
    ms = {k: [] for k in recs}
    for _ in range(args.steps):
        for name, rec in recs.items():
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            res[name] = rec.beam_search_many(inputs, raise_on_failure=False)
            torch.cuda.synchronize(dev)
            ms[name].append((time.perf_counter() - t0) * 1e3)
    out = {"gpu": bench.gpu_identity(0), "workload": "configs[2]: %d utterances x <= %d frames, beam %d, WSJ architecture"
           % (case["U"], case["T"], case["beam"]), "lm": {"states": S, "arcs": num_arcs, "weight": 0.5,
                                                          "no_transition_cost": 20.0}}
    for name in recs:
        med = sorted(ms[name])[len(ms[name]) // 2]
        found = [r for r in res[name] if r is not None]
        out[name] = {"ms_per_batch_median": round(med, 1), "utterances_per_s": round(case["U"] / (med * 1e-3), 2),
                     "decoded": len(found),
                     "mean_best_length": round(float(np.mean([len(r[0][0]) for r in found])), 1) if found else 0.0}
    out["fusion_overhead"] = round(out["no_lm"]["ms_per_batch_median"] and
                                   (out["lm"]["ms_per_batch_median"] / out["no_lm"]["ms_per_batch_median"] - 1.0), 4)
    # the LM kernels alone: per-class CUDA events in a run of their own
    tot, cnt = C.c_double(), C.c_int64()
    lib.lvsr_profile_read(b"lm", C.byref(tot), C.byref(cnt))
    lib.lvsr_profile_enable(1)
    recs["lm"].beam_search_many(inputs, raise_on_failure=False)
    torch.cuda.synchronize(dev)
    lib.lvsr_profile_enable(0)
    lib.lvsr_profile_read(b"lm", C.byref(tot), C.byref(cnt))
    out["lm"]["lm_kernel_launches"] = int(cnt.value)
    out["lm"]["lm_kernel_us_per_launch"] = round(tot.value * 1e3 / max(1, cnt.value), 1)
    for cls in ("gemm", "bigru", "attention", "window", "dense", "readout"):
        lib.lvsr_profile_read(cls.encode(), C.byref(tot), C.byref(cnt))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
