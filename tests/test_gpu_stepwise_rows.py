"""The step-wise decoder (attention.cu window_kernel / att_step_kernel, decoder.cu) at the row counts and encoded lengths
where it carries the work, compared with the float64 oracle element by element.

The persistent decoder (dec_scan.cu) runs a teacher-forced cost of at most 64 rows at the WSJ decoder width (C = 256).
Everything else runs on the step-wise kernels: every beam search, every greedy step of `generate`, and every cost or
training forward of more than 64 rows.  The attention step gives each row a cluster of cs CTAs.  attention_step picks
the largest cs that keeps R * cs * 2 within the SMs (one wave), then doubles cs while a CTA's share of the row,
ceil(T'/cs) positions, does not fit in 227 KB of shared memory; a T' that 8 CTAs cannot hold is refused with an error.
The expected cs of every case is derived here from the device's SM count and a restatement of att_smem_floats /
att_red_floats (attention_row.cuh), never written as a literal.  At the decoder widths of bench.NET (E = M = 512,
K = 10 filters of 2 * 100 + 1 taps) one CTA holds 1288 positions with location attention and 3119 with content
attention, clusters of 2 hold 2546, of 8 hold 9480.

Each case asserts through SpeechRecognizer.decoder_plan() the decoder that ran and the attention step's cluster size,
and compares with the oracle at the bounds and with the helpers of test_gpu_attention_plans.py (weights relative per
element, exactly 0 outside the window; energies over their scale; costs, states, weighted averages and
log-probabilities per element with a floor of 0.1 of their scale).  Beam searches must give the oracle's best
hypothesis and every finished hypothesis, reordered only between costs within 1e-4 (test_gpu_widths.py).

Worst errors measured over every case of this file on an H100 80GB HBM3 (700 W power limit), against the bounds of
test_gpu_attention_plans.py: weights 1.3e-5 (5e-5), energies 2.2e-6 (2e-5), weight sums 2.1e-7 (2e-6), costs 1.9e-6
(1e-5), log-probabilities 1.4e-6 (2e-6, the greedy steps at T' = 2000), states 4.4e-5 and weighted averages 2.4e-5
(1e-4), search costs 4.1e-6 (1e-5), gradients 3.3e-6 of each parameter's largest entry (1e-4).  Most of the file's
3.5 minutes on that machine are the oracle's.
"""
import numpy as np
import pytest

import content_oracle as CO
from helpers import O, WSJ, check_energies, check_grads, check_weights, elementwise_err, f32, make_recognizer
from test_gpu_attention_plans import TOL, WSUM_TOL, _compare, _inputs, _make_content, _params, _set_env
from test_gpu_widths import _peaky, _same_up_to_near_ties

pytestmark = pytest.mark.gpu

# the decoder widths of bench.NET on one unsubsampled BiGRU(256) layer: E = 512, T' = T, so T' is chosen freely
ARCH = dict(num_features=40, dims_bidir=[256], subsample=[1], dim_dec=256, dim_matcher=512, conv_n=100,
            conv_num_filters=10, num_phonemes=63, post_merge_dims=[256], maxout_pieces=2)

FULL = dict(type="expanding", initial_begin=0, initial_end=100000, min_speed=0, max_speed=0)
NARROW = dict(type="expanding", initial_begin=0, initial_end=20, min_speed=3.0, max_speed=9.0)
MEDIAN = dict(type="window_around_median", before=20, after=24)
MEAN = dict(type="window_around_mean", before=16, after=16)
STRESS = dict(type="window_around_median", before=100, after=100)       # bench.py configs[4]
PRIORS = dict(full=FULL, narrow=NARROW, median=MEDIAN, mean=MEAN, stress=STRESS)

# ---- the cluster size attention_step must choose --------------------------------------------------------------------

SMEM_MAX = 227 * 1024        # dynamic shared memory one CTA may opt in to
ATT_NW = 16                  # warps of an attention CTA (ATT_NT = 512 threads)


def _smem_bytes(Tp, cs, loc=True, M=512, E=512, K=10, n=100, wh_rows=16):
    """att_smem_floats in bytes for a chunk of ceil(T'/cs) positions, with a handler copy of wh_rows rows (16: padded,
    K: compact)."""
    tc = -(-Tp // cs)
    f = 2 * M                                                        # sq, sv
    if loc:
        f += wh_rows * M + (2 * n + 1) * (12 if K <= 12 else 16)       # sWh, sfiltT
        f += tc + 2 * n + 8 + (tc + 16) * 16                         # salpha, sF
    f += 2 * (tc + 16) + 96                                          # se, su, block scratch
    f += max(8 * E, ATT_NW * (tc + 16))                              # sred (att_red_floats)
    f += cs * 4 + cs * E + 32                                        # xs, xctx, tail
    return 4 * f


def _longest_row(cs, loc=True, **widths):
    """The largest T' a cluster of cs CTAs holds: the largest multiple of cs whose chunk fits.  `widths`: M, E, K, n
    of _smem_bytes (bench.NET's by default)."""
    lo, hi = 1, 1 << 20
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if _smem_bytes(mid * cs, cs, loc, **widths) <= SMEM_MAX else (lo, mid - 1)
    return lo * cs


def _sms():
    import torch
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _expected_cs(R, Tp, loc=True, **widths):
    cs = 1
    while cs < 8 and R * cs * 2 <= _sms() and -(-Tp // (cs * 2)) >= 16:
        cs *= 2
    while cs < 8 and _smem_bytes(Tp, cs, loc, **widths) > SMEM_MAX and -(-Tp // (cs * 2)) >= 16:
        cs *= 2
    return cs


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


_RECS = {}


def _model(prior=None, content=False):
    """One recognizer per prior (and one for content attention) for the whole file."""
    key = "content" if content else prior
    if key not in _RECS:
        if content:
            cfg = CO.make_config(**ARCH)
            params = _params(cfg, seed=5, content=True)
            _RECS[key] = (cfg, params, _make_content(cfg, params))
        else:
            cfg = O.make_config(prior=PRIORS[prior], **ARCH)
            params = _params(cfg, seed=5)
            _RECS[key] = (cfg, params, make_recognizer(cfg, params))
    return _RECS[key]


def _cost_case(monkeypatch, what, prior, B, Tp, L, seed, content=False):
    """cost_matrix on given attended arrays -> the plan that ran, after the element-by-element comparison."""
    torch = _torch()
    cfg, params, rec = _model(prior, content)
    att, attm, labels, lm = inputs = _inputs(cfg, B, Tp, L, seed=seed)
    _set_env(monkeypatch)
    got = rec.cost_matrix(labels, lm, torch.as_tensor(att, dtype=torch.float32, device="cuda"),
                          torch.as_tensor(attm, dtype=torch.float32, device="cuda"), return_all=True)
    plan = rec.decoder_plan()
    print("PLAN", what, B, Tp, prior, {k: plan[k] for k in ("ran", "kernel", "cs", "att_cs")})
    want = (CO if content else O).cost_matrix(cfg, params, *inputs, return_all=True)
    _compare(got, want, content, "%s B=%d T'=%d %s" % (what, B, Tp, prior))
    return plan


def _assert_stepwise(plan, R, Tp, loc=True):
    assert not plan["ran"] and plan["kernel"] == "stepwise", plan
    assert plan["att_cs"] == _expected_cs(R, Tp, loc), (R, Tp, plan)


def test_the_derived_limits_are_consistent():
    """The restated footprint grows with the chunk, and each larger cluster holds a longer row."""
    _torch()
    rows = [_longest_row(cs) for cs in (1, 2, 4, 8)]
    assert rows == sorted(rows) and len(set(rows)) == 4, rows
    assert _longest_row(1, loc=False) >= 2000                # the content case below runs in one CTA
    for cs, Tp in zip((1, 2, 4, 8), rows):
        assert _smem_bytes(Tp, cs) <= SMEM_MAX < _smem_bytes(Tp + cs, cs)
    print("longest rows at cs 1, 2, 4, 8:", rows, "content:", _longest_row(1, loc=False), "SMs:", _sms())


# ---- row counts around the persistent decoder's limit ---------------------------------------------------------------

# (B, prior): 64 rows is the persistent decoder's last batch; 65 and 66 rows run step-wise at the one-wave cs of a
# 132-SM part (2), from 67 rows on at cs 1; every prior at 67 rows
ROWS = [(64, "full"), (64, "median"), (65, "narrow"), (65, "mean"), (66, "full"), (66, "median"), (67, "full"),
        (67, "narrow"), (67, "median"), (67, "mean"), (128, "narrow"), (128, "mean")]


@pytest.mark.parametrize("B,prior", ROWS, ids=["%d-%s" % c for c in ROWS])
def test_cost_matrix_rows_around_the_cliff(B, prior, monkeypatch):
    Tp = 150 + B % 50
    plan = _cost_case(monkeypatch, "rows", prior, B, Tp, 10, seed=B)
    if B <= 64:
        assert plan["ran"] and plan["kernel"] == "dec_scan", plan
    else:
        _assert_stepwise(plan, B, Tp)


# ---- long alignments on the step kernel -----------------------------------------------------------------------------

LONG = [("cs1_limit", "stress"), ("cs1_limit_plus_1", "stress"), ("cs1_limit_plus_1", "full"), ("t2000", "stress"),
        ("t2000", "full")]


@pytest.mark.parametrize("where,prior", LONG, ids=["%s-%s" % c for c in LONG])
def test_long_rows_on_the_step_kernel(where, prior, monkeypatch):
    """72 rows (cs 1 by the one-wave rule) at the longest row one CTA holds, one position more and T' = 2000: the last
    two need clusters of 2.  The full window is the oracle's slowest case, so it runs at the two longer rows only."""
    Tp = dict(cs1_limit=_longest_row(1), cs1_limit_plus_1=_longest_row(1) + 1, t2000=2000)[where]
    plan = _cost_case(monkeypatch, where, prior, 72, Tp, 4, seed=Tp)
    _assert_stepwise(plan, 72, Tp)
    assert plan["att_cs"] == (1 if where == "cs1_limit" else 2), plan


def test_long_rows_content_attention(monkeypatch):
    """Content attention needs no location features: 72 rows of T' = 2000 in one CTA each."""
    plan = _cost_case(monkeypatch, "content", None, 72, 2000, 5, seed=9, content=True)
    _assert_stepwise(plan, 72, 2000, loc=False)
    assert plan["att_cs"] == 1, plan


def test_greedy_steps_at_scale(monkeypatch):
    """logprobs_computer / next_state_computer, the path of generate, for 72 rows of T' = 2000."""
    torch = _torch()
    cfg, params, rec = _model("stress")
    R, Tp = 72, 2000
    att, attm, _, _ = _inputs(cfg, R, Tp, 1, seed=31)
    _set_env(monkeypatch)
    ctx = dict(attended=torch.as_tensor(att, dtype=torch.float32, device="cuda"),
               attended_mask=torch.as_tensor(attm, dtype=torch.float32, device="cuda"))
    st_o = O.initial_states(cfg, params, R, att)
    st_g = rec._initial_states(Tp, R)
    for step in range(3):
        lp_o = O.logprobs_computer(cfg, params, att, attm, st_o)
        lp_g = rec._logprobs(ctx, st_g).double().cpu().numpy()
        _assert_stepwise(rec.decoder_plan(), R, Tp)
        errs = dict(logprobs=elementwise_err(lp_g, lp_o))
        y = lp_o.argmin(axis=1)
        st_o = O.next_state_computer(cfg, params, att, attm, st_o, y)
        st_g = rec._next_states(ctx, st_g, y)
        g = {k: v.double().cpu().numpy() for k, v in st_g.items()}
        check_weights(g["weights"], st_o["weights"], errs)
        check_energies(g["energies"], st_o["energies"], errs)
        errs["states"] = elementwise_err(g["states"], st_o["states"])
        errs["weighted_averages"] = elementwise_err(g["weighted_averages"], st_o["weighted_averages"])
        print("ERRS greedy step", step, " ".join("%s=%.2e" % kv for kv in sorted(errs.items())))
        for k, e in errs.items():
            assert e <= (WSUM_TOL if k.endswith("_sum") else TOL[k]), (step, k, e)
        assert np.array_equal(g["step"], st_o["step"])


# ---- batched beam search --------------------------------------------------------------------------------------------

def _search_matches_oracle(cfg, params, rec, utts, beam, scale, compare):
    """search_many over all `utts` together; the first `compare` of them against O.beam_search one by one."""
    rec.init_beam_search(beam)
    got = rec._beam_search.search_many([u.astype(np.float32) for u in utts], cfg["eos_label"],
                                       [int(u.shape[0] / scale) for u in utts], raise_on_failure=False)
    n_found = n_hyp = 0
    for u, g in zip(utts[:compare], got):
        try:
            want = O.beam_search(cfg, params, u, beam)
        except O.CandidateNotFoundError:
            assert g is None
            continue
        assert g is not None and g[0][0] == want[0][0], (g, want)        # the best hypothesis
        n_hyp += _same_up_to_near_ties(g, want)
        n_found += 1
    print("utterances with a result:", n_found, "finished hypotheses compared:", n_hyp)
    assert n_found >= compare // 2 and n_hyp > n_found       # some utterance finished several hypotheses
    return rec.decoder_plan()


@pytest.mark.parametrize("prior", ["stress", "expanding"])
def test_search_many_long_utterances(prior):
    """8 utterances of 1300-1500 frames at beam 10: 8 rows at the first step (cs 8), then up to 80 rows, which one
    CTA per row cannot hold at these lengths."""
    _torch()
    scale = 100.0
    pri = STRESS if prior == "stress" else dict(type="expanding", initial_begin=0, initial_end=100, min_speed=5.0,
                                                max_speed=60.0)
    cfg = O.make_config(prior=pri, max_decoded_length_scale=scale, **ARCH)
    params = _peaky(cfg, 81, gain=4.0, eos_bias=2.0)
    rng = np.random.RandomState(82)
    utts = [f32(rng.normal(size=(T, cfg["num_features"]))) for T in rng.randint(1300, 1501, size=8)]
    assert min(u.shape[0] for u in utts) > _longest_row(1)
    plan = _search_matches_oracle(cfg, params, make_recognizer(cfg, params), utts, 10, scale,
                                  compare=8 if prior == "stress" else 4)
    assert plan["att_cs"] >= 2, plan                     # no step of these lengths fits in one CTA per row


def test_search_many_wsj_width():
    """The shape of bench.py's configs[2]: 32 utterances of at most 800 frames (T' <= 200) at beam 10, all decoded
    together; 8 of them compared with the oracle."""
    _torch()
    scale = 8.0
    cfg = O.make_config(max_decoded_length_scale=scale, **WSJ)
    params = _peaky(cfg, 91, gain=4.0, eos_bias=2.0)
    rng = np.random.RandomState(92)
    lens = rng.randint(480, 801, size=32)
    lens[0] = 800
    utts = [f32(rng.normal(size=(T, cfg["num_features"]))) for T in lens]
    rec = make_recognizer(cfg, params)
    plan = _search_matches_oracle(cfg, params, rec, utts, 10, scale, compare=8)
    assert not plan["ran"] and plan["att_cs"] >= 1, plan


# ---- training forward past 64 rows ----------------------------------------------------------------------------------

def test_gradients_at_67_rows(monkeypatch):
    _torch()
    _set_env(monkeypatch)
    cfg = O.make_config(prior=MEDIAN, **dict(ARCH, num_phonemes=32))
    params = O.init_params(cfg, seed=41, scale=10.0)
    batch = O.synthetic_batch(cfg, B=67, T=24, seed=42)
    _, rec = check_grads(cfg, params, batch)
    _assert_stepwise(rec.decoder_plan(), 67, 24)


# ---- a row no cluster holds -----------------------------------------------------------------------------------------

def test_row_longer_than_any_cluster_is_refused(monkeypatch):
    """One position more than 8 CTAs hold is refused before any launch; the recognizer then computes as before."""
    torch = _torch()
    cfg, params, rec = _model("stress")
    _set_env(monkeypatch)

    def logprobs(Tp):
        att, attm, _, _ = _inputs(cfg, 2, Tp, 1, seed=51, lens=[Tp, Tp])
        ctx = dict(attended=torch.as_tensor(att, dtype=torch.float32, device="cuda"),
                   attended_mask=torch.as_tensor(attm, dtype=torch.float32, device="cuda"))
        return rec._logprobs(ctx, rec._initial_states(Tp, 2)).cpu()

    before = logprobs(300)
    with pytest.raises(RuntimeError, match="shared memory"):
        logprobs(_longest_row(8) + 1)
    after = logprobs(300)
    assert torch.equal(before, after)
