"""Generate tests/golden/bench_train_golden.npz: the float64 gradient oracle (oracle/lvsr_oracle_grad.py) of the
training step bench.py times (`--mode train`): TRAIN_WORKLOAD (64 utterances of up to 1500 frames, 190 label steps) on
bench.NET with bench.init_values weights and the inputs of bench.train_bench's first shard.

The oracle's autograd tape cannot hold the whole batch, so the gradient is built one utterance at a time.  The batch
cost is sum(costs) / B; under the default prior every utterance attends its whole encoded sequence, a padded frame
leaves the masked GRU state unchanged and a padded label costs 0, so the batch gradient is exactly the mean of the
gradients of the utterances cropped to their own frames and labels and run with B = 1 (tests/test_bench_train_golden_cpu.py
checks this on small configs).  A window prior cuts one window for the whole batch, so the generator refuses any other.

The readout's maxout has a kink wherever its two pieces tie, and over the 12,160 label rows of this batch twenty of its
128 units come within 2e-5 of one at some row (the smallest gap is below 1e-6).  A float32 forward can take the other
piece there, which moves that row's whole backward; one such flip costs several times the gradient bar.  So the oracle
runs with the zero bias of the first piece of each such unit offset by a multiple of KINK_EPS / 4 that puts every row
of the unit at least KINK_EPS from its kink (kink_nudges), and the test applies the same offsets.

Stored (kept small; the inputs are regenerated from their seeds and pinned by SHA-256 digests):
    meta            JSON: workload, net, train_conf, seed
    batch_sha256    digests of recordings, recordings_mask, labels, labels_mask as bench.synthetic_batch returns them
    params_sha256   digest of the float32 initial parameters, in parameter order (before the offsets)
    kink_eps, nudge_index, nudge_value
                    the offsets: post_merge/bias.b[nudge_index] += nudge_value (float32)
    min_gap_before, min_gap
                    the smallest |first piece - second piece| over label-unmasked rows without and with the offsets
    cost, costs     the mean cost and the float64 cost matrix [L, B]
    grad_norm       L2 norm of the mean gradient
    names, stats    per parameter: sum g, sum |g|, max |g|, sum g^2, and g . r_j for 4 N(0,1) vectors r_j (projections())
    entry_offsets, entry_index, entry_value
                    entries of each parameter's gradient (flat index, value): every entry of a parameter of at most
                    FULL_MAX entries; otherwise its TOP largest |g| and SAMPLED more from RandomState(SAMPLE_SEED)

Run from the repo root (about 5 minutes on 8 CPU cores):
    python tests/golden/make_bench_train_golden.py [--workers N] [--out PATH]
"""
import argparse
import hashlib
import json
import multiprocessing
import os
import sys
import time
from collections import OrderedDict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from oracle import lvsr_oracle as O  # noqa: E402

PATH = os.path.join(ROOT, "tests", "golden", "bench_train_golden.npz")
SEED = bench.shard_seed(0, base=4321)          # bench.train_bench's inputs on rank 0
NPROJ, PROJ_SEED = 4, 11
FULL_MAX, TOP, SAMPLED, SAMPLE_SEED = 4096, 128, 384, 13
STAT_NAMES = ("sum", "sum_abs", "max_abs", "sum_sq") + tuple("proj%d" % j for j in range(NPROJ))
KINK_EPS = 2e-5                 # as tests/helpers.py: above the float32 error of a readout pre-activation on the GPU
_RO = "/recognizer/generator/readout"


def bench_inputs():
    """(cfg, (recordings, recordings_mask, labels, labels_mask), float32 params) exactly as bench.train_bench builds
    them; params in O.param_shapes order."""
    cfg = O.make_config(**bench.NET)
    params = bench.init_values(O.param_shapes(cfg))
    batch = bench.synthetic_batch(**bench.TRAIN_WORKLOAD, seed=SEED)
    return cfg, batch, params


def digest(a):
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(("%s%s" % (a.dtype.str, a.shape)).encode())
    h.update(a.tobytes())
    return h.hexdigest()


def batch_digests(batch):
    return [digest(a) for a in batch]


def params_digest(params):
    h = hashlib.sha256()
    for k, v in params.items():
        h.update(k.encode())
        h.update(digest(np.asarray(v, dtype=np.float32)).encode())
    return h.hexdigest()


def check_prior(cfg):
    """The per-utterance decomposition needs every utterance to attend its whole encoded sequence."""
    if cfg["prior"] != O.DEFAULT_PRIOR:
        raise ValueError("the batch gradient is a mean of per-utterance gradients only under the default prior, "
                         "not %r" % (cfg["prior"],))


def crop(batch, b):
    """Utterance b of a padded batch, cropped to its own frames and labels, as a batch of one."""
    x, m, labels, lm = batch
    T, L = int(np.asarray(m)[:, b].sum()), int(np.asarray(lm)[:, b].sum())
    return x[:T, b:b + 1], m[:T, b:b + 1], labels[:L, b:b + 1], lm[:L, b:b + 1]


_WORK = {}


def _init_worker(cfg, params, batch, oracle=None):
    import torch
    torch.set_num_threads(1)           # one utterance is too small for threads to help; the workers share the cores
    _WORK.update(cfg=cfg, params=params, batch=batch, oracle=oracle)


def _oracles():
    """(gradient oracle, forward oracle) of the model: oracle/lvsr_oracle{_grad}.py, or the importable module named by
    `oracle` (one that has both cost_and_grads and recognizer_cost, e.g. tests/unidirectional_oracle.py)."""
    if _WORK.get("oracle") is None:
        from oracle import lvsr_oracle_grad as G
        return G, O
    import importlib
    mod = importlib.import_module(_WORK["oracle"])
    return mod, mod


def _utterance(b):
    G, _ = _oracles()
    cost, grads, costs = G.cost_and_grads(_WORK["cfg"], _WORK["params"], *crop(_WORK["batch"], b), return_costs=True)
    return cost, grads, costs[:, 0]


def _readout_preactivations(b):
    """float64 readout pre-activations [L_b, post_merge_dim] of utterance b (what the maxout reduces)."""
    cfg, p = _WORK["cfg"], _WORK["params"]
    p64 = {k: np.asarray(v, dtype=np.float64) for k, v in p.items()}
    x, m, labels, lm = crop(_WORK["batch"], b)
    out = _oracles()[1].recognizer_cost(cfg, p64, x.astype(np.float64), m.astype(np.float64), labels, lm.astype(np.float64),
                            return_all=True)
    pre = out["weighted_averages"] @ p64[_RO + "/merge/transform_weighted_averages.W"] + p64[_RO + "/post_merge/bias.b"]
    if cfg["use_states_for_readout"]:
        pre = pre + out["states"] @ p64[_RO + "/merge/transform_states.W"]      # states = s_{i-1}
    return pre[:, 0]


def _pool(cfg, params, batch, workers, oracle=None):
    if workers > 1:
        return multiprocessing.get_context("spawn").Pool(workers, initializer=_init_worker,
                                                         initargs=(cfg, params, batch, oracle))
    _WORK.update(cfg=cfg, params=params, batch=batch, oracle=oracle)
    return None


def _map(pool, fn, items):
    return pool.imap(fn, items) if pool is not None else map(fn, items)


def maxout_gaps(cfg, params, batch, workers=1, oracle=None):
    """float64 (first piece - second piece) of every two-piece maxout unit of the readout at every label-unmasked
    row, [n_rows, units]; oracle: as _oracles."""
    assert cfg["post_merge_activation"] == "maxout" and cfg["maxout_pieces"] == 2, cfg
    pool = _pool(cfg, params, batch, workers, oracle)
    try:
        pre = np.concatenate(list(_map(pool, _readout_preactivations, range(np.asarray(batch[2]).shape[1]))))
    finally:
        if pool is not None:
            pool.close()
            pool.join()
    return pre[:, 0::2] - pre[:, 1::2]


def kink_nudges(gaps, eps=KINK_EPS):
    """Offsets of the first piece's bias (post_merge/bias.b) of every unit with a row whose two pieces lie within eps
    of each other: the smallest multiple of eps / 4 that moves every row of the unit at least eps from its kink.  The
    derivative of a maxout jumps where its pieces tie, and a float32 forward may take either piece there; the
    readout's pre-activations feed nothing back into the teacher-forced decoder, so the offset moves each gap by
    exactly itself.  -> {unit: offset}, float32 offsets."""
    out = {}
    for j in np.flatnonzero((np.abs(gaps) < eps).any(axis=0)):
        for step in range(1, 401):
            d = [np.float32(s * step * eps / 4) for s in (1, -1)]
            ok = [dd for dd in d if np.abs(gaps[:, j] + float(dd)).min() >= eps]
            if ok:
                out[int(j)] = ok[0]
                break
        else:
            raise RuntimeError("no bias offset of unit %d clears every kink" % j)
    return out


def apply_nudges(params, index, value):
    """params with post_merge/bias.b[index] += value (the fixture's kink offsets)."""
    out = OrderedDict(params)
    b = np.array(out[_RO + "/post_merge/bias.b"], dtype=np.float32)
    b[np.asarray(index, dtype=np.int64)] += np.asarray(value, dtype=np.float32)
    out[_RO + "/post_merge/bias.b"] = b
    return out


def mean_of_utterance_grads(cfg, params, batch, workers=1, oracle=None):
    """float64 (sum(costs) / B, costs [L, B], gradient) of the batch, as the mean over its utterances run one at a time.
    Summed in utterance order, so the result does not depend on `workers`; oracle: as _oracles."""
    check_prior(cfg)
    L, B = np.asarray(batch[2]).shape
    costs = np.zeros((L, B))
    total, grads = 0.0, None
    pool = _pool(cfg, params, batch, workers, oracle)
    try:
        for b, (cost, g, c) in enumerate(_map(pool, _utterance, range(B))):
            total += cost
            costs[:len(c), b] = c
            if grads is None:
                grads = OrderedDict((k, v.copy()) for k, v in g.items())
            else:
                for k in grads:
                    grads[k] += g[k]
    finally:
        if pool is not None:
            pool.close()
            pool.join()
    return total / B, costs, OrderedDict((k, v / B) for k, v in grads.items())


def projections(shape, rng):
    return rng.normal(size=(NPROJ,) + tuple(shape))


def grad_stats(grads):
    """[n_params, len(STAT_NAMES)] in parameter order; projection vectors drawn from RandomState(PROJ_SEED) in that order."""
    rng = np.random.RandomState(PROJ_SEED)
    rows = []
    for g in grads.values():
        g = np.asarray(g, dtype=np.float64)
        r = projections(g.shape, rng)
        rows.append([g.sum(), np.abs(g).sum(), np.abs(g).max(), (g * g).sum()] +
                    [(g * r[j]).sum() for j in range(NPROJ)])
    return np.array(rows)


def entry_indices(grads):
    """Flat indices stored for each parameter: all of a small one; the TOP largest |g| and SAMPLED others of a large one."""
    rng = np.random.RandomState(SAMPLE_SEED)
    out = []
    for g in grads.values():
        a = np.abs(np.asarray(g, dtype=np.float64)).ravel()
        if a.size <= FULL_MAX:
            out.append(np.arange(a.size))
            continue
        top = np.argsort(-a, kind="stable")[:TOP]
        rest = np.setdiff1d(np.arange(a.size), top)
        out.append(np.concatenate([top, np.sort(rng.choice(rest, SAMPLED, replace=False))]))
    return out


def reduce_grads(grads):
    idx = entry_indices(grads)
    offsets = np.cumsum([0] + [len(i) for i in idx])
    values = np.concatenate([np.asarray(g, dtype=np.float64).ravel()[i] for g, i in zip(grads.values(), idx)])
    return dict(names=np.array(list(grads)), stats=grad_stats(grads), entry_offsets=offsets.astype(np.int64),
                entry_index=np.concatenate(idx).astype(np.int64), entry_value=values)


def meta():
    return dict(workload=bench.TRAIN_WORKLOAD, net=bench.NET, train_conf=bench.TRAIN_CONF, seed=SEED)


def write_fixture(out, cfg, batch, params, meta, workers, oracle=None):
    """The fixture of the training step of (cfg, params) on `batch` (the fields listed above) -> `out`; oracle: as
    _oracles."""
    t0 = time.time()
    check_prior(cfg)
    gaps = maxout_gaps(cfg, params, batch, workers=workers, oracle=oracle)
    nudges = kink_nudges(gaps)
    index = np.array([2 * j for j in sorted(nudges)], dtype=np.int64)             # the unit's first piece
    value = np.array([nudges[j] for j in sorted(nudges)], dtype=np.float32)
    moved = gaps.copy()
    moved[:, index // 2] += value.astype(np.float64)
    assert np.abs(moved).min() >= KINK_EPS
    cost, costs, grads = mean_of_utterance_grads(cfg, apply_nudges(params, index, value), batch, workers=workers,
                                                 oracle=oracle)
    norm = float(np.sqrt(sum((g * g).sum() for g in grads.values())))
    np.savez_compressed(out, meta=np.array(json.dumps(meta, sort_keys=True)),
                        batch_sha256=np.array(batch_digests(batch)), params_sha256=np.array(params_digest(params)),
                        kink_eps=np.float64(KINK_EPS), nudge_index=index, nudge_value=value,
                        min_gap_before=np.float64(np.abs(gaps).min()), min_gap=np.float64(np.abs(moved).min()),
                        cost=np.float64(cost), costs=costs, grad_norm=np.float64(norm), **reduce_grads(grads))
    print("oracle %.0f s, %d maxout units moved off their kinks, cost %.6f, |g| %.6f -> %s (%.0f KB)" % (
        time.time() - t0, len(index), cost, norm, out, os.path.getsize(out) / 1024))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workers", type=int, default=min(8, os.cpu_count() or 1))
    ap.add_argument("--out", default=PATH)
    args = ap.parse_args()
    cfg, batch, params = bench_inputs()
    write_fixture(args.out, cfg, batch, params, meta(), args.workers)


if __name__ == "__main__":
    main()
