"""The long-utterance workload bench.py --mode stress times (configs[4]: bench.STRESS_NET, 16 utterances x 2000 frames,
3 x BiGRU(256) without subsampling, so T' = 2000; 63 symbols; window_around_median(100, 100); 60 label steps), compared
with the float64 oracle, and the persistent decoder at that shape under alignments that keep every rank of its clusters
busy.

At these widths (E = M = 512, C = 256, K = 10 filters of 201 taps) the planner's one-wave start is cs 8 (16 rows x 4 x 2
<= 132 SMs), whose islands fit in shared memory but need 16 co-resident 8-CTA clusters; where the device holds fewer,
the plan is 4-CTA islands, which fit only with the compact handler copy (wh_rows = K): chunks of tc_cap = 500
positions, grid 64, ncg 64, nc1/nc2/nc3 = 24/8/8, the dense tiles' scratch in the attention scratch (red_alias).  cs 1
and 2 do not fit.  Every plan is restated here from derive() (test_gpu_encoded_widths._derive with the handler rows as
an argument) and the occupancy query's answers the planner reports, never written as literals.  A cluster splits each
step's window cut evenly over its ranks (attention_row: ceil(Tw / cs) positions each), so every rank works at every step
and the cases choose windows from 100 positions up to the whole utterance: ranks end their share on partial 16-position
P tiles, and the merge of max, sum and partial context and the location convolution's halo cross rank boundaries.

  1. The benchmark itself, end to end: bench.init_values parameters, bench.synthetic_batch inputs at rank 0's seed,
     encode + cost_matrix, and the host entry rec.cost that --mode stress also times, on the same plan.  Bound:
     test_gpu_metric.py's 1e-4 relative (max |got - want| / max |want|) per quantity; the alignment's argmax equal
     wherever the oracle's top two weights differ by more than 1e-4; weights exactly 0 outside the window and at masked
     positions.  From the oracle's weights: every rank owns positions at every step, some steps end on partial P tiles,
     and ranks other than 0 own the median.
  2. The decoder alone on the oracle's encoder output (rounded to float32), under five more priors, at the per-element
     bounds of test_gpu_attention_plans.py (_compare): a window sweeping over the utterance, one growing to all of it
     (P and H exceed the L2: the evict-first instantiation, bit-identical to LVSR_DEC_L2=off), the full window,
     window_around_mean, and window_around_median with an alignment the location term moves along the utterance
     (_moving).  Each case asserts from the oracle's weights the coverage it claims.
  3. The sweeping case under every plan switch: default, LVSR_DEC_LAYOUT=global, LVSR_DEC_CS=8 (declined unless the
     device holds 16 eight-CTA clusters), LVSR_DEC_CS=1 and 2 (declined), LVSR_NO_DEC_SCAN=1 (the step-wise kernels at
     the attention step's cluster size).

Worst errors, their bounds and the file's runtime on an H100 are in DESIGN.md §2.
"""
import numpy as np
import pytest

import bench
from helpers import O, f32, make_recognizer, rel_err
from test_gpu_attention_plans import _compare, _set_env
from test_gpu_dec_l2 import _expected_kb, _l2_bytes
from test_gpu_encoded_widths import DS_ROWS, _derive
from test_gpu_stepwise_rows import SMEM_MAX, _expected_cs, _sms

pytestmark = pytest.mark.gpu

W = bench.STRESS_WORKLOAD
NET = bench.STRESS_NET
E, C, M, K, N = 2 * NET["dims_bidir"][-1], NET["dim_dec"], NET["dim_matcher"], NET["conv_num_filters"], NET["conv_n"]
TOL = 1e-4                        # test_gpu_metric.py's bound for the benchmarked shapes
TIE = 1e-4                        # top two weights closer than this: the argmax may differ

STRESS = dict(type="window_around_median", before=100, after=100)           # stress_bench's prior
SWEEP = dict(type="expanding", initial_begin=0, initial_end=100, min_speed=30, max_speed=35)
GROW = dict(type="expanding", initial_begin=0, initial_end=100, min_speed=0, max_speed=35)
FULL = dict(type="expanding", initial_begin=0, initial_end=100000, min_speed=0, max_speed=0)
MEAN = dict(type="window_around_mean", before=100, after=100)
PRIORS = dict(stress=STRESS, sweep=SWEEP, grow=GROW, full=FULL, mean=MEAN, moving=STRESS)

_ATT = "/recognizer/generator/att_trans/conv_att"
_CACHE = {}


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _cached(key, fn):
    if key not in _CACHE:
        _CACHE[key] = fn()
    return _CACHE[key]


def _batch():
    """stress_bench's inputs on rank 0"""
    return _cached("batch", lambda: bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"],
                                                          seed=bench.shard_seed(0, base=777)))


def _bench_params():
    """bench.init_values over the recognizer's parameter shapes, as stress_bench sets them (float32)"""
    def make():
        rec = make_recognizer(O.make_config(prior=STRESS, **NET))
        return {k: v.astype(np.float64) for k, v in bench.init_values(rec.parameter_shapes()).items()}
    return _cached("params", make)


def _moving(params):
    """An alignment that the location term moves along the utterance: filter 0 has 61 unit taps 20 to 80 positions back
    (F[t] = the previous alignment's mass over [t - 80, t - 20]), handler row 0 points along the energy vector, so a
    position's energy rises with that mass, and the content term is scaled by 0.05.  The drive is weak on purpose: the
    handler product's 3-term bf16 split carries about 2^-17 of the location term, and a location term of a few units of
    energy (a 5-tap filter with 4x the gain moved 35 positions a step) put weight errors of 1e-4 to 1e-3 on both
    decoders.  Here the location term stays near one unit and the median advances about 25 positions a step."""
    p = dict(params)
    filt = p[_ATT + "/conv1d.filters"].copy()
    filt[0] = 0.0
    filt[0, N + 20:N + 81] = 1.0
    wh = p[_ATT + "/handler.W"].copy()
    v = p[_ATT + "/energy_comp/linear.W"][:, 0]
    wh[0] = 0.04 * v / np.abs(v).mean()
    p[_ATT + "/conv1d.filters"], p[_ATT + "/handler.W"] = f32(filt), f32(wh)
    for k in ("/preprocess.W", "/state_trans/transform_states.W"):
        p[_ATT + k] = f32(p[_ATT + k] * 0.05)
    return p


def _model(case):
    """(oracle config, float32 parameters in float64, recognizer) of a case; one recognizer per case"""
    def make():
        cfg = O.make_config(prior=PRIORS[case], **NET)
        params = _moving(_bench_params()) if case == "moving" else _bench_params()
        rec = make_recognizer(cfg)
        rec.set_parameter_values({k: v.astype(np.float32) for k, v in params.items()})
        return cfg, params, rec
    return _cached(("model", case), make)


def _oracle_encoder():
    """the oracle's encoder output on the float32 inputs, and its mask"""
    def make():
        cfg, params, _ = _model("stress")
        x, m, _, _ = _batch()
        return O.encoder(cfg, params, x.astype(np.float64), m.astype(np.float64))
    return _cached("encoder", make)


def _oracle_cost(case):
    """the oracle's cost_matrix(return_all=True): on its own encoder output for the benchmark, on that output rounded to
    float32 (what the decoder-only cases feed the GPU) for the others"""
    def make():
        cfg, params, _ = _model(case)
        att, attm = _oracle_encoder()
        _, _, labels, lm = _batch()
        return O.cost_matrix(cfg, params, att if case == "stress" else f32(att), attm, labels, lm.astype(np.float64),
                             return_all=True)
    return _cached(("cost", case), make)


# ---- the plan, restated from dec_scan.cu plan_and_launch / derive ----------------------------------------------------

def _fit(Tp, cs, ncg):
    """derive()'s handler choice: the padded copy (16 rows) if it fits, else the compact one (K rows).
    -> (nc1, nc2, nc3, bytes, red_alias, wh_rows), or None when neither fits"""
    for rows in (16, K):
        d = _derive(E, C, M, Tp, cs, ncg, True, K=K, n=N, wh_rows=rows)
        if d is not None and d[3] <= SMEM_MAX:
            return d + (rows,)
    return None


def _restated_plan(B, Tp, clusters, cs=None, layout=None):
    """The plan plan_and_launch chooses for B rows of T' positions under LVSR_DEC_CS = cs and LVSR_DEC_LAYOUT = layout;
    None: declined, the step-wise kernels run.  clusters[c]: the occupancy query's answer for clusters of c CTAs (how
    many are co-resident), asked for every candidate whose tiles fit."""
    sms, nrg = _sms(), -(-B // DS_ROWS)
    c = 1
    while c < 8 and B * c * 2 <= sms and -(-Tp // (c * 2)) >= 16:      # the one-wave start
        c *= 2
    if cs is not None:
        if cs > 1 and -(-Tp // cs) < 16:
            return None
        c = cs
    for c in (c, c // 2, c // 4, c // 8):
        if c < 1 or (cs is not None and c != cs):
            return None
        islands = B >= DS_ROWS and layout != "global"
        if layout == "islands" and not islands:
            return None
        G = B * c if islands else sms // c * c
        d = _fit(Tp, c, B // nrg * c if islands else G // nrg)
        if d is None and islands and layout != "islands":
            islands, G = False, sms // c * c
            d = _fit(Tp, c, G // nrg)
        if d is None:
            continue
        assert c in clusters, ("no occupancy answer for clusters of %d CTAs" % c, clusters)
        if clusters[c] * c < G:
            if islands:
                continue                              # islands need one co-resident cluster per row
            G = clusters[c] * c
            shrunk = _fit(Tp, c, G // nrg)
            if G < c or shrunk is None or shrunk[5] != d[5]:
                continue
            d = shrunk
        if B * c > G:
            continue
        return dict(cs=c, nisl=nrg if islands else 0, nrg=1 if islands else nrg, grid=G,
                    ncg=B // nrg * c if islands else G // nrg, nc1=d[0], nc2=d[1], nc3=d[2], tc_cap=-(-Tp // c),
                    red_alias=int(d[4]), wh_rows=d[5], kernel="dec_scan<COMPACT>" if d[5] != 16 else "dec_scan")
    return None


def _cs8_clusters(case):
    """The occupancy query's answer for the 8-CTA candidate, the planner's first at this shape: a run of `case`'s model
    (the same kernel instantiation, with or without the L2 hints) forced to 8-CTA clusters, in an environment of its own
    that is restored when it returns.  The query runs on the device, so the restated plan below confirms the planner's
    arithmetic given the answers; that 15 or 16 clusters are co-resident is the device's to say."""
    def ask():
        with pytest.MonkeyPatch.context() as mp:
            _, plan = _decoder_run(mp, case, "cs 8 occupancy", LVSR_DEC_CS="8")
        return plan["max_clusters"]
    return _cached(("cs8_clusters", case), ask)


def _check_plan(plan, Tp, what, cs8_clusters, cs=None, layout=None):
    """The plan that ran is the restated one; returns it (None: the planner declined and the step-wise kernels ran).
    cs8_clusters: _cs8_clusters of the case."""
    clusters = {8: cs8_clusters}
    if plan["ran"] or cs is not None:
        clusters[plan["cs"] or cs] = plan["max_clusters"]          # the last answer: the candidate that ran, or cs
    want = _restated_plan(W["B"], Tp, clusters, cs, layout)
    print("PLAN", what, {k: v for k, v in plan.items() if not k.startswith("_")}, "restated:", want,
          "co-resident clusters:", clusters)
    if want is None:
        assert not plan["ran"] and plan["kernel"] == "stepwise" and plan["cs"] == 0, (what, plan)
        return None
    assert plan["ran"], (what, plan, want)
    for k, v in want.items():
        assert plan[k] == v, (what, k, plan, want)
    return want


# ---- 1. the benchmark, whole path ------------------------------------------------------------------------------------

def test_bench_stress_matches_oracle(monkeypatch):
    torch = _torch()
    cfg, params, rec = _model("stress")
    x, m, labels, lm = _batch()
    want_att, want_attm = _oracle_encoder()
    want = _oracle_cost("stress")
    cs8 = _cs8_clusters("stress")
    _set_env(monkeypatch)                     # LVSR_DEC_CHECK=1: launch status 0 and every hand-over word written
    att, attm = rec.encode(x, m)
    got = rec.cost_matrix(labels, lm, att, attm, return_all=True)
    assert rec.launch_status() == (0, 0)
    Tp = att.shape[0]
    assert tuple(att.shape) == (W["T"], W["B"], E) and np.array_equal(attm.cpu().numpy(), want_attm)
    plan = _check_plan(rec.decoder_plan(), Tp, "bench", cs8)
    # the compact handler at cs 4 in islands; the padded copy does not fit at cs 4
    assert plan is not None and plan["kernel"] == "dec_scan<COMPACT>" and plan["wh_rows"] == K, plan
    assert _derive(E, C, M, Tp, plan["cs"], plan["ncg"], True, K=K, n=N)[3] > SMEM_MAX
    g = {k: v.double().cpu().numpy() for k, v in got.items()}
    errs = dict(attended=rel_err(att.double().cpu().numpy(), want_att))
    for k in ("costs", "states", "weighted_averages", "weights", "energies"):
        errs[k] = rel_err(g[k], want[k])
    print("ERRS bench", " ".join("%s=%.2e" % kv for kv in sorted(errs.items())))
    for k, e in errs.items():
        assert e < TOL, (k, e)
    w, ww = g["weights"], want["weights"]
    top2 = np.sort(ww, axis=-1)[..., -2:]
    clear = top2[..., 1] - top2[..., 0] > TIE
    print("near ties:", int((~clear).sum()), "of", clear.size)
    assert np.array_equal(w.argmax(-1)[clear], ww.argmax(-1)[clear])
    # exactly 0 outside the window (the oracle's zeros) and at masked positions; at most before + after + 1 positions
    assert not np.any(w[ww == 0]) and not np.any(g["energies"][want["energies"] == 0])
    assert not np.any(w * (1 - want_attm.T[None]))
    assert (w > 0).sum(-1).max() <= STRESS["before"] + STRESS["after"] + 1
    _median_coverage(cfg, ww, plan["cs"], "bench")
    # the host-buffer entry point --mode stress also times, on the same plan
    host = rec.cost(x, m, labels, lm)
    assert rec.launch_status() == (0, 0)
    assert rel_err(host, want["costs"]) < TOL, rel_err(host, want["costs"])
    after = rec.decoder_plan()
    assert all(after[k] == v for k, v in plan.items()), (after, plan)


# ---- 2. every rank at work, decoder only -----------------------------------------------------------------------------

def _decoder_run(monkeypatch, case, what, **env):
    """cost_matrix of `case` on the oracle's float32 attended under the env switches -> (outputs, plan)"""
    torch = _torch()
    _, _, rec = _model(case)
    att, attm = _oracle_encoder()
    _, _, labels, lm = _batch()
    _set_env(monkeypatch)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    got = rec.cost_matrix(labels, lm, torch.as_tensor(att, dtype=torch.float32, device="cuda"),
                          torch.as_tensor(attm, dtype=torch.float32, device="cuda"), return_all=True)
    assert rec.launch_status() == (0, 0), what
    return got, rec.decoder_plan()


def _lengths():
    return _oracle_encoder()[1].sum(0).astype(int)


def _extents(w):
    """[L, B, 2]: first and last position of non-zero weight per (step, row); -1 for rows without any"""
    nz = w > 0
    first = np.where(nz.any(-1), nz.argmax(-1), -1)
    last = np.where(nz.any(-1), w.shape[-1] - 1 - nz[..., ::-1].argmax(-1), -1)
    return np.stack([first, last], -1)


def _coverage(case, w):
    """Assert, from the oracle's weights, the coverage the case exists for."""
    lens, L, Tp = _lengths(), w.shape[0], w.shape[2]
    ext = _extents(w)
    steps = np.arange(L)[:, None]
    if case == "sweep":
        # windows [30 i, 100 + 35 i): up to position 1999; rows whose utterance ends before the window holds nothing
        assert ext[..., 1].max() == Tp - 1
        past = np.minimum(30 * steps, Tp - 1) >= lens[None, :]
        assert past.any() and np.array_equal(ext[..., 0] < 0, past), (past.sum(), (ext[..., 0] < 0).sum())
        print("sweep: (step, row) pairs past the utterance's end:", int(past.sum()))
    elif case == "grow":
        # [0, 100 + 35 i): the last steps cover every row's whole utterance
        assert np.all(ext[-1, :, 0] == 0) and np.array_equal(ext[-1, :, 1], lens - 1)
    elif case == "mean":
        # window_around_mean: the cut follows the alignment's mean past the first window
        assert ext[..., 1].max() > 2 * MEAN["after"], ext[..., 1].max()
    elif case == "moving":
        # the alignment advances about 25 positions a step: windows hold 500 and 1000 at some step
        for pos in (500, 1000):
            assert np.any((ext[..., 0] <= pos) & (ext[..., 1] >= pos)), pos
        med = (np.cumsum(w, -1) >= 0.5).argmax(-1)
        step = np.diff(med[:20], axis=0)
        print("moving: median advance per step over the first 20 steps %d..%d (median %d), largest weight %.3f"
              % (step.min(), step.max(), np.median(step), w.max()))
        assert 15 <= np.median(step) <= 40, step
    elif case == "full":
        assert np.array_equal(ext[..., 0], np.zeros_like(ext[..., 0]))
        assert np.array_equal(ext[..., 1], np.broadcast_to(lens - 1, ext[..., 1].shape))


def _median_coverage(cfg, w, cs, what):
    """From the oracle's weights [L, B, T'] under a window-around-median prior: each step's window cut (attention_window
    on the previous alignment), its split over cs ranks (ceil(Tw / cs) positions each, attention_row), and the rank that
    owns the median of each new alignment (the first with mass up to 0.5).  Asserts that every rank owns positions at
    every step, that some steps end the ranks' shares on partial 16-position P tiles, and that ranks other than 0 own
    the median; returns the owners [L, B] (-1: a row without mass)."""
    L, B, Tp = w.shape
    prev = np.zeros((B, Tp))
    prev[:, 0] = 1.0                                      # initial_glimpses: one-hot at position 0
    owners, shares = np.full((L, B), -1), []
    for i in range(L):
        b0, b1, _ = O.attention_window(cfg, Tp, prev, np.full(B, i))
        tc = -(-(b1 - b0) // cs)
        shares.append(tc)
        assert (cs - 1) * tc < b1 - b0, (what, i, b0, b1, cs)      # the last rank owns positions too
        mass = np.cumsum(w[i, :, b0:b1], axis=-1)
        for b in range(B):
            if mass[b, -1] > 0.5:
                owners[i, b] = int(np.argmax(mass[b] >= 0.5)) // tc
        prev = w[i]
    shares = np.array(shares)
    counts = [int((owners == r).sum()) for r in range(cs)]
    print("%s: positions per rank %d..%d, median owners per rank %s" % (what, shares.min(), shares.max(), counts))
    assert np.any(shares % 16), (what, shares)
    assert sum(counts[1:]) > 0, (what, counts)
    return owners


def _widest_window(prior, Tp, L):
    """dec_scan.cu l2_plan: the most positions one step of the expanding prior reads (None for the other priors)"""
    if prior["type"] != "expanding":
        return None
    i = np.arange(L)
    b = np.floor(np.clip(prior["initial_begin"] + i * prior["min_speed"], 0, Tp - 1))
    e = np.ceil(np.clip(prior["initial_end"] + i * prior["max_speed"], 0, Tp))
    return int((e - b).max())


@pytest.mark.parametrize("case", ["sweep", "grow", "full", "mean", "moving"])
def test_every_rank_matches_oracle(case, monkeypatch):
    torch = _torch()
    want = _oracle_cost(case)
    _coverage(case, want["weights"])
    cs8 = _cs8_clusters(case)
    got, plan = _decoder_run(monkeypatch, case, case)
    Tp = want["weights"].shape[2]
    ran = _check_plan(plan, Tp, case, cs8)
    if case == "moving":
        _median_coverage(_model(case)[0], want["weights"], ran["cs"], case)
    _compare(got, want, False, case)
    # the evict-first loads: on under the expanding prior when one step's P and H over its widest window exceed the L2
    widest = _widest_window(PRIORS[case], Tp, want["weights"].shape[0])
    over = widest is not None and widest * W["B"] * (M + E) * 4 > _l2_bytes(torch)
    if widest is not None and over:
        assert plan["l2_evict_first_kb"] == _expected_kb(torch, widest, W["B"], M, E) > 0, plan
    else:
        assert plan["l2_evict_first_kb"] == 0, plan
    if case == "grow":
        assert over, "the growing window must run the evict-first instantiation"
        off, plan_off = _decoder_run(monkeypatch, case, "grow L2 off", LVSR_DEC_L2="off")
        assert plan_off["l2_evict_first_kb"] == 0 and plan_off["kernel"] == plan["kernel"], plan_off
        for k in ("costs", "weights", "energies", "states", "weighted_averages"):
            assert torch.equal(got[k], off[k]), k


# ---- 3. every plan this shape can take -------------------------------------------------------------------------------

SWITCHES = [("default", {}, None, None),
            ("global", dict(LVSR_DEC_LAYOUT="global"), None, "global"),
            ("cs8", dict(LVSR_DEC_CS="8"), 8, None),
            ("cs1", dict(LVSR_DEC_CS="1"), 1, None),
            ("cs2", dict(LVSR_DEC_CS="2"), 2, None),
            ("no_dec_scan", dict(LVSR_NO_DEC_SCAN="1"), None, None)]


@pytest.mark.parametrize("name,env,cs,layout", SWITCHES, ids=[s[0] for s in SWITCHES])
def test_sweeping_window_under_every_plan(name, env, cs, layout, monkeypatch):
    _torch()
    want = _oracle_cost("sweep")
    cs8 = _cs8_clusters("sweep")
    got, plan = _decoder_run(monkeypatch, "sweep", name, **env)
    Tp = want["weights"].shape[2]
    if name == "no_dec_scan":
        print("PLAN", name, plan)
        assert not plan["ran"] and plan["kernel"] == "stepwise", plan
        assert plan["att_cs"] == _expected_cs(W["B"], Tp), plan
    else:
        ran = _check_plan(plan, Tp, name, cs8, cs, layout)
        if name in ("cs1", "cs2"):
            assert ran is None and _fit(Tp, cs, W["B"] * cs) is None, plan       # no handler copy fits
        elif name == "cs8":
            # the tiles fit; whether the plan runs is the occupancy query's answer
            assert _fit(Tp, 8, W["B"] * 8) is not None
            assert (ran is not None) == (plan["max_clusters"] >= W["B"]), plan
        else:
            assert ran is not None and (ran["nisl"] == 0) == (layout == "global"), plan
    _compare(got, want, False, name)
