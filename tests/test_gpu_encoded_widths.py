"""The decoder side at every encoded width E = 2 * dims_bidir[-1] the encoder gives (128, 384, 640, 768, 896, 1024;
256 and 512 are the other files'), compared with the float64 oracle element by element, and the training step at the
encoder widths and weight-gradient products the other files never train.

The kernels split their work by E: attention_row's partial weighted average into E / 4 column groups and
min(8, 512 / (E / 4)) position groups (8 with half the threads idle at E = 128, 5 at 384, 3 at 640, 2 from 768 on), the
attention step's shared memory by 8E (sred) and cs * E (xctx) floats, the persistent decoder's gate product by E + C
(dec_scan.cu kper_ok: 256 = 128 + 128 is KPER 8 across the [context | state] boundary, 512 = 384 + 128, 768 = 384 + 384
or 640 + 128; from E = 768 on no C gives a KPER shape and every cost runs step-wise).  Each decoder case builds one
unsubsampled BiGRU(E / 2) layer and hands `attended` to the decoder directly, as test_gpu_attention_plans.py does, so the
oracle never runs the encoder there.  Every case asserts the plan it targets through decoder_plan() / encoder_plan():

  * teacher-forced costs at every E with two priors and content attention, B = 6, T' = 40: the persistent decoder where
    kper_ok(E + C) and kper_ok(C) hold, with cs, ncg, nc1, nc2, nc3 and the shared-memory fit restated from derive()
    (_derive below), and the step-wise kernels under LVSR_NO_DEC_SCAN=1 with the cluster size attention_step must pick;
  * LVSR_DEC_CS = 1, 2, 4, 8 at E = 128 and 384 (C = 128), global (B = 6) and islands (B = 16; 8-CTA islands are not
    co-resident on an H100, as test_gpu_attention_plans.py shows), and LVSR_ATT_CS = 1 and 8 at E = 1024;
  * the attention step's length cliffs at E = 768 and 1024 (bench.NET's decoder widths), from the footprint restated in
    test_gpu_stepwise_rows.py: the longest row at cs 1 and one position more (72 rows), the longest row at cs 8 (2 rows),
    and one position more refused with the attention-step error, after which the same handle decodes as before;
  * six greedy steps at E = 128, 896, 1024; search_many token for token against O.beam_search at E = 384 and 896 under
    both stop criteria and at E = 1024 with content attention, every finished hypothesis compared;
  * gradients (helpers.check_grads) at [448] with B = 33, T = 63 (2079 rows: FFMA weight gradients, 448 % 128 != 0, and a
    partial 4-row group), the same under LVSR_NO_TC_GEMM=1, [384] at the same shape (tensor-core weight gradients over a
    contraction padded to 2080), [192] alone, the pyramid [192, 448], content attention at E = 896; two optimizer steps
    (helpers.train_like_the_oracle) at 448.

The bounds are those of test_gpu_attention_plans.py (TOL, WSUM_TOL), except the greedy steps' log-probabilities and the
search costs, held to test_gpu_widths.py's (4e-6, 1e-5), and check_grads' 1e-4 for the gradients.  Worst errors measured
over every case of this file on an H100 80GB HBM3 (700 W power limit): weights 2.0e-5 (bound 5e-5), energies 3.7e-6
(2e-5), weight sums 1.7e-7 (2e-6), costs 1.7e-6 (1e-5), states 6.3e-5 and weighted averages 4.3e-5 (1e-4), log-probabilities
3.5e-6 (4e-6; 72 rows at E = 1024), search costs 2.9e-6 (1e-5), gradients 2.6e-5 of a parameter's largest entry (1e-4).
The file runs in about 65 s there; most of it is the oracle's, chiefly the four 72-row cliff cases (7-9 s each).
"""
import numpy as np
import pytest

import content_oracle as CO
from helpers import O, check_energies, check_grads, check_weights, elementwise_err, f32, make_recognizer
from helpers import train_like_the_oracle
from oracle import lvsr_oracle_grad as G
from test_gpu_attention_plans import (PRIORS, TOL, WSUM_TOL, _case, _compare, _inputs, _make_content, _params,
                                      _set_env, _tp)
from test_gpu_stepwise_rows import ATT_NW, SMEM_MAX, STRESS, _expected_cs, _longest_row, _smem_bytes, _sms
from test_gpu_widths import TOL as WIDTHS_TOL, _peaky, _same_up_to_near_ties

pytestmark = pytest.mark.gpu

# log-probabilities of the greedy steps at test_gpu_widths.py's bound (4e-6): the readout contracts the weighted average
# over E, and at 72 rows of E = 1024 their error measured 3.5e-6 (1.4e-6 at E = 512, test_gpu_stepwise_rows.py)
STEP_TOL = dict(TOL, logprobs=WIDTHS_TOL["logprobs"])


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _arch(E, C=128, M=256, n=8):
    return dict(num_features=40, dims_bidir=[E // 2], subsample=[1], dim_dec=C, dim_matcher=M, conv_n=n,
                conv_num_filters=10, num_phonemes=32, post_merge_dims=[128], maxout_pieces=2)


def _config(E, C=128, prior="median", **kw):
    """prior None: content attention."""
    if prior is None:
        return CO.make_config(**_arch(E, C), **kw)
    return O.make_config(prior=PRIORS[prior], **_arch(E, C), **kw)


def _recognizer(cfg, params):
    return _make_content(cfg, params) if cfg["attention_type"] == "content" else make_recognizer(cfg, params)


# ---- the persistent decoder's planner, restated (dec_scan.cu) -------------------------------------------------------

DS_ROWS = 16             # rows per dense tile
DS_WARPS = 16            # warps of a persistent-decoder CTA


def _kper_ok(k):
    return k % 128 == 0 and k // 32 in (4, 8, 12, 16, 24)


def _derive(E, C, M, Tp, cs, ncg, loc, K=10, n=8, wh_rows=16):
    """derive() with a handler copy of wh_rows rows (16: padded, K: compact): (nc1, nc2, nc3, dynamic shared memory in
    bytes, red_alias); None: no tile fits."""
    r8 = lambda x: (x + 7) // 8 * 8
    nc2 = r8(-(-C // ncg))
    nc1, nc3 = 3 * nc2, r8(-(-M // ncg))
    if max(nc1, nc2, nc3) > 24:
        return None
    tc = -(-Tp // cs)
    red_f = DS_WARPS * DS_ROWS * max(nc1, nc2, nc3)
    red_alias = max(8 * E, ATT_NW * (tc + 16)) >= red_f
    f = _smem_bytes(Tp, cs, loc, M=M, E=E, K=K, n=n, wh_rows=wh_rows) // 4
    f = (f + 3) // 4 * 4 + (E + C) * (nc1 + 4) + C * (nc2 + 4) + C * (nc3 + 4)
    f = (f + 3) // 4 * 4 + 3 * DS_ROWS * nc2 + 4 + (0 if red_alias else red_f)
    return nc1, nc2, nc3, 4 * f + 64, red_alias


def _one_wave_cs(R, Tp):
    cs = 1
    while cs < 8 and R * cs * 2 <= _sms() and -(-Tp // (cs * 2)) >= 16:
        cs *= 2
    return cs


def _check_derived_tiles(plan, E, C, M, B, loc, what):
    """The tile widths the planner reported are derive()'s for the CTAs per row group it reported, and they fit."""
    nrg = 1 if plan["nisl"] else -(-B // DS_ROWS)
    assert plan["ncg"] == (B // plan["nisl"] * plan["cs"] if plan["nisl"] else plan["grid"] // nrg), (what, plan)
    d = _derive(E, C, M, plan["_Tp"], plan["cs"], plan["ncg"], loc)
    assert d is not None and d[3] <= SMEM_MAX, (what, d, plan)
    assert (plan["nc1"], plan["nc2"], plan["nc3"]) == d[:3], (what, d, plan)


# ---- teacher-forced costs at every encoded width --------------------------------------------------------------------

# (E, C, prior or None for content attention); the persistent decoder's pairs are (128, 128), (128, 256), (384, 128),
# (384, 384), (640, 128)
COSTS = [(128, 128, "median"), (128, 256, "mean"), (128, 128, None),
         (384, 128, "narrow"), (384, 384, "median"), (384, 384, None),
         (640, 128, "mean"), (640, 128, "full"), (640, 128, None),
         (768, 128, "median"), (768, 256, "mean"), (768, 128, None),
         (896, 128, "narrow"), (896, 128, "median"), (896, 128, None),
         (1024, 128, "full"), (1024, 256, "mean"), (1024, 128, None)]


def _cost(monkeypatch, cfg, params, inputs, want, what, **env):
    torch = _torch()
    att, attm, labels, lm = inputs
    rec = _recognizer(cfg, params)
    _set_env(monkeypatch, att_cs=env.pop("att_cs", None))
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    got = rec.cost_matrix(labels, lm, torch.as_tensor(att, dtype=torch.float32, device="cuda"),
                          torch.as_tensor(attm, dtype=torch.float32, device="cuda"), return_all=True)
    plan = rec.decoder_plan()
    plan["_Tp"] = att.shape[0]
    print("PLAN", what, {k: v for k, v in plan.items() if not k.startswith("_")})
    assert rec.launch_status() == (0, 0)
    _compare(got, want, cfg["attention_type"] == "content", what)
    return plan


@pytest.mark.parametrize("E,C,prior", COSTS, ids=["E%d-C%d-%s" % (E, C, p or "content") for E, C, p in COSTS])
def test_cost_matrix_matches_oracle(E, C, prior, monkeypatch):
    """The planner's own choice, then the step-wise kernels on the same inputs."""
    loc, B, Tp, M = prior is not None, 6, 40, 256
    cfg = _config(E, C, prior)
    params = _params(cfg, seed=E + C, content=not loc)
    inputs = _inputs(cfg, B, Tp, 7, seed=E // 64 + C)
    want = (O if loc else CO).cost_matrix(cfg, params, *inputs, return_all=True)
    what = "E=%d C=%d %s" % (E, C, prior or "content")
    plan = _cost(monkeypatch, cfg, params, inputs, want, what)
    cs = _one_wave_cs(B, Tp)
    if _kper_ok(E + C) and _kper_ok(C):
        # the planner's first candidate: cs CTAs per row, one global row group on every SM
        first = _derive(E, C, M, Tp, cs, _sms() // cs * cs, loc)
        assert first is not None and first[3] <= SMEM_MAX, (what, first)
        assert plan["ran"], ("the persistent decoder fits (derive: nc1, nc2, nc3, bytes = %s) but was declined"
                             % (first,), what, plan)
        assert plan["kernel"] == ("dec_scan" if loc else "dec_content") and plan["cs"] == cs, (what, plan)
        assert plan["nisl"] == 0 and plan["nrg"] == 1, (what, plan)
        _check_derived_tiles(plan, E, C, M, B, loc, what)
    else:
        assert E >= 768, (E, C)                 # E + C = 896 to 1280: no KPER shape
        assert not plan["ran"] and plan["kernel"] == "stepwise", (what, plan)
    plan = _cost(monkeypatch, cfg, params, inputs, want, what + " step-wise", LVSR_NO_DEC_SCAN="1")
    assert not plan["ran"] and plan["kernel"] == "stepwise", (what, plan)
    assert plan["att_cs"] == _expected_cs(B, Tp, loc, M=M, E=E, n=8), (what, plan)


# ---- forced cluster sizes ------------------------------------------------------------------------------------------

FORCED = [(E, cs, layout) for E in (128, 384) for cs in (1, 2, 4, 8) for layout in ("global", "islands")
          if (cs, layout) != (8, "islands")]
_ROTATE = ("median", "mean", "narrow", "full")


@pytest.mark.parametrize("E,cs,layout", FORCED, ids=["E%d-cs%d-%s" % c for c in FORCED])
def test_forced_persistent_plans_match_oracle(E, cs, layout, monkeypatch):
    B = 16 if layout == "islands" else 6
    prior = _ROTATE[(cs.bit_length() + E // 128) % 4]
    cfg = _config(E, 128, prior)
    params = _params(cfg, seed=E + cs)
    inputs = _inputs(cfg, B, _tp(cs), 6, seed=E + 10 * cs + B)
    plan = _case(monkeypatch, "E=%d forced cs %d %s %s" % (E, cs, layout, prior), cfg, params, inputs, cs=cs,
                 layout=layout)
    _check_derived_tiles(plan, E, 128, 256, B, True, "E=%d cs %d %s" % (E, cs, layout))


@pytest.mark.parametrize("cs", [1, 8])
def test_forced_attention_step_at_e1024(cs, monkeypatch):
    """E + C = 1152: the cost runs on the step-wise kernels, at the forced attention-step cluster size."""
    cfg = _config(1024, 128, "median")
    params = _params(cfg, seed=cs)
    inputs = _inputs(cfg, 6, _tp(cs), 6, seed=cs + 3)
    want = O.cost_matrix(cfg, params, *inputs, return_all=True)
    plan = _cost(monkeypatch, cfg, params, inputs, want, "E=1024 att_cs %d" % cs, att_cs=cs)
    assert not plan["ran"] and plan["kernel"] == "stepwise" and plan["att_cs"] == cs, plan


# ---- greedy steps and the attention step's length cliffs -----------------------------------------------------------

def _greedy(monkeypatch, cfg, params, rec, att, attm, steps, what, widths):
    """`steps` logprobs_computer / next_state_computer steps against the oracle; the attention step's cluster size
    must be _expected_cs's at every step."""
    torch = _torch()
    R, Tp = att.shape[1], att.shape[0]
    _set_env(monkeypatch)
    ctx = dict(attended=torch.as_tensor(att, dtype=torch.float32, device="cuda"),
               attended_mask=torch.as_tensor(attm, dtype=torch.float32, device="cuda"))
    st_o = O.initial_states(cfg, params, R, att)
    st_g = rec._initial_states(Tp, R)
    cs = set()
    for step in range(steps):
        lp_o = O.logprobs_computer(cfg, params, att, attm, st_o)
        lp_g = rec._logprobs(ctx, st_g).double().cpu().numpy()
        cs.add(rec.decoder_plan()["att_cs"])
        errs = dict(logprobs=elementwise_err(lp_g, lp_o))
        y = lp_o.argmin(axis=1)
        st_o = O.next_state_computer(cfg, params, att, attm, st_o, y)
        st_g = rec._next_states(ctx, st_g, y)
        cs.add(rec.decoder_plan()["att_cs"])
        g = {k: v.double().cpu().numpy() for k, v in st_g.items()}
        check_weights(g["weights"], st_o["weights"], errs)
        check_energies(g["energies"], st_o["energies"], errs)
        errs["states"] = elementwise_err(g["states"], st_o["states"])
        errs["weighted_averages"] = elementwise_err(g["weighted_averages"], st_o["weighted_averages"])
        print("\nERRS", what, "step", step, " ".join("%s=%.2e" % kv for kv in sorted(errs.items())))
        for k, e in errs.items():
            assert e <= (WSUM_TOL if k.endswith("_sum") else STEP_TOL[k]), (what, step, k, e)
        assert np.array_equal(g["step"], st_o["step"])
    assert cs == {_expected_cs(R, Tp, True, **widths)}, (what, cs)
    return cs.pop()


@pytest.mark.parametrize("E", [128, 896, 1024])
def test_greedy_steps_match_oracle(E, monkeypatch):
    cfg = _config(E, 128, "median")
    params = _params(cfg, seed=E + 1)
    Tp = 40
    att, attm, _, _ = _inputs(cfg, 3, Tp, 1, seed=E, lens=[Tp, Tp - 4, Tp - 9])
    _greedy(monkeypatch, cfg, params, make_recognizer(cfg, params), att, attm, 6, "greedy E=%d" % E,
            dict(M=256, E=E, n=8))


# bench.NET's decoder widths (M = 512, C = 256, 10 filters of 201 taps) under its stress prior, at which
# test_gpu_stepwise_rows.py's footprint restatement holds by default
_CLIFF_ARCH = dict(num_features=40, subsample=[1], dim_dec=256, dim_matcher=512, conv_n=100, conv_num_filters=10,
                   num_phonemes=63, post_merge_dims=[256], maxout_pieces=2)
_CLIFF_RECS = {}


def _cliff_model(E):
    if E not in _CLIFF_RECS:
        cfg = O.make_config(prior=STRESS, dims_bidir=[E // 2], **_CLIFF_ARCH)
        params = _params(cfg, seed=E // 64)
        _CLIFF_RECS[E] = (cfg, params, make_recognizer(cfg, params))
    return _CLIFF_RECS[E]


CLIFFS = [(E, where) for E in (768, 1024) for where in ("cs1_limit", "cs1_limit_plus_1", "cs8_limit")]


@pytest.mark.parametrize("E,where", CLIFFS, ids=["E%d-%s" % c for c in CLIFFS])
def test_attention_step_length_cliffs(E, where, monkeypatch):
    """72 rows (cs 1 by the one-wave rule) at the longest row one CTA holds at this E and one position more (clusters
    of 2); 2 rows at the longest row 8 CTAs hold."""
    cfg, params, rec = _cliff_model(E)
    limit = dict(cs1_limit=_longest_row(1, E=E), cs1_limit_plus_1=_longest_row(1, E=E) + 1,
                 cs8_limit=_longest_row(8, E=E))[where]
    R = 2 if where == "cs8_limit" else 72
    att, attm, _, _ = _inputs(cfg, R, limit, 1, seed=limit)
    cs = _greedy(monkeypatch, cfg, params, rec, att, attm, 2, "E=%d %s T'=%d" % (E, where, limit), dict(E=E))
    assert cs == dict(cs1_limit=1, cs1_limit_plus_1=2, cs8_limit=8)[where], (E, where, limit, cs)


@pytest.mark.parametrize("E", [768, 1024])
def test_row_longer_than_any_cluster_is_refused(E, monkeypatch):
    """One position more than 8 CTAs hold at this E is refused before any launch; the handle then decodes a valid row
    as the oracle does."""
    torch = _torch()
    cfg, params, rec = _cliff_model(E)
    _set_env(monkeypatch)
    Tp = _longest_row(8, E=E) + 1
    assert _smem_bytes(Tp, 8, E=E) > SMEM_MAX >= _smem_bytes(Tp - 1, 8, E=E)
    att, attm, _, _ = _inputs(cfg, 2, Tp, 1, seed=E, lens=[Tp, Tp])
    ctx = dict(attended=torch.as_tensor(att, dtype=torch.float32, device="cuda"),
               attended_mask=torch.as_tensor(attm, dtype=torch.float32, device="cuda"))
    with pytest.raises(RuntimeError, match="attention_step: T'=%d positions do not fit in shared memory" % Tp):
        rec._logprobs(ctx, rec._initial_states(Tp, 2))
    att, attm, _, _ = _inputs(cfg, 3, 300, 1, seed=E + 1)
    _greedy(monkeypatch, cfg, params, rec, att, attm, 2, "E=%d after the refusal" % E, dict(E=E))


# ---- search --------------------------------------------------------------------------------------------------------

# (E, prior or None for content attention, readout gain, eos bias): chosen so that every utterance finishes
# hypotheses of several lengths
SEARCH = [(384, "median", 4.0, 4.0), (896, "mean", 4.0, 4.0), (1024, None, 4.0, 4.0)]


@pytest.mark.parametrize("E,prior,gain,eos_bias", SEARCH, ids=["E%d-%s" % (c[0], c[1] or "content") for c in SEARCH])
@pytest.mark.parametrize("stop_on,char_discount", [("patience", 0.0), ("optimistic_future_cost", 0.1)])
def test_search_many_matches_oracle(E, prior, gain, eos_bias, stop_on, char_discount):
    """search_many over three utterances at beam 5: the oracle's best hypothesis and every finished one."""
    _torch()
    scale, beam = 2.0, 5
    cfg = _config(E, 128, prior, max_decoded_length_scale=scale)
    params = _peaky(cfg, E + 41, gain=gain, eos_bias=eos_bias)
    rng = np.random.RandomState(E)
    utts = [f32(rng.normal(size=(T, cfg["num_features"]))) for T in (36, 25, 30)]
    rec = _recognizer(cfg, params)
    rec.init_beam_search(beam)
    got = rec._beam_search.search_many([u.astype(np.float32) for u in utts], cfg["eos_label"],
                                       [int(u.shape[0] / scale) for u in utts], raise_on_failure=False,
                                       stop_on=stop_on, char_discount=char_discount)
    n_found = n_hyp = 0
    for u, g in zip(utts, got):
        want = (O if prior else CO).beam_search(cfg, params, u, beam, stop_on=stop_on, char_discount=char_discount)
        assert g is not None and g[0][0] == want[0][0], (g, want)          # the best hypothesis
        n_hyp += _same_up_to_near_ties(g, want)
        n_found += 1
    plan = rec.decoder_plan()
    print("E=%d %s: finished hypotheses compared: %d" % (E, stop_on, n_hyp), plan)
    assert n_found == len(utts) and n_hyp > n_found, n_hyp           # some utterance finished several hypotheses
    assert not plan["ran"] and plan["att_cs"] >= 1, plan
    assert rec.encoder_plan()[0]["cs"] == E // 64, rec.encoder_plan()


# ---- training ------------------------------------------------------------------------------------------------------

GRADS = {                 # name -> (widths, subsampling, B, T, attention)
    "d448_2079_rows": ([448], [1], 33, 63, "content_and_conv"),
    "d384_tc_2079_rows": ([384], [1], 33, 63, "content_and_conv"),
    "d192": ([192], [1], 4, 40, "content_and_conv"),
    "pyramid_192_448": ([192, 448], [1, 2], 5, 41, "content_and_conv"),
    "d448_content": ([448], [1], 4, 32, "content"),
}


@pytest.mark.parametrize("case,no_tc", [(c, False) for c in sorted(GRADS)] + [("d448_2079_rows", True)],
                         ids=sorted(GRADS) + ["d448_2079_rows-no_tc"])
def test_gradients_match_oracle(case, no_tc, monkeypatch):
    _torch()
    _set_env(monkeypatch)
    if no_tc:
        monkeypatch.setenv("LVSR_NO_TC_GEMM", "1")
    dims, sub, B, T, attention = GRADS[case]
    M = CO if attention == "content" else O
    cfg = M.make_config(**dict(_arch(2 * dims[-1]), dims_bidir=dims, subsample=sub))
    params = {k: f32(v) for k, v in M.init_params(cfg, seed=len(case), scale=10.0).items()}
    x, m, labels, lm = O.synthetic_batch(cfg, B=B, T=T, seed=B + T)
    _, rec = check_grads(cfg, params, (f32(x), m, labels, lm))
    plan = rec.encoder_plan()
    print(case, no_tc, [(p["bwd_cs"], p["wgrad"], p["wgrad_kpad"], p["T"]) for p in plan], rec.decoder_plan())
    Tl = T
    for l, p in enumerate(plan):
        assert p["bwd_cs"] == dims[l] // 32 and p["tape"] and p["T"] == Tl, (l, p)
        tc = not no_tc and Tl * B >= 2048 and dims[l] % 128 == 0
        assert (p["wgrad"], p["wgrad_kpad"]) == (("tc", -(-Tl * B // 32) * 32) if tc else ("ffma", 0)), (l, p)
        Tl = -(-Tl // sub[l])
    if case.startswith("d448"):
        assert plan[0]["bwd_cs"] == 14 and plan[0]["wgrad"] == "ffma"
    if case == "d384_tc_2079_rows":
        assert (plan[0]["wgrad"], plan[0]["wgrad_kpad"]) == ("tc", 2080), plan


def test_two_optimizer_steps_at_448(monkeypatch):
    _torch()
    _set_env(monkeypatch)
    cfg = O.make_config(prior=PRIORS["median"], **_arch(896))
    params = O.init_params(cfg, seed=448, scale=10.0)
    tc = G.make_train_config(gradient_threshold=2.0, rules=("momentum", "adadelta"), scale=0.05, momentum=0.5,
                             decay_rate=0.95, epsilon=1e-6, max_norm=1.0)
    rec, _, _ = train_like_the_oracle(cfg, params, tc, B=4, T=32)
    p = rec.encoder_plan()[0]
    assert p["bwd_cs"] == 14 and p["tape"] and p["wgrad"] == "ffma", p
