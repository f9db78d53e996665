"""Every plan the decoder planners can choose, forced one at a time and compared with the float64 oracle element by
element.

How a row is computed is decided at run time (dec_scan.cu plan_and_launch / derive, attention.cu attention_step): the
cluster size cs, island or global layout, the padded or compact handler copy, whether the dense scratch aliases the
attention scratch.  The shapes other tests use reach only a few of these plans, and a plan that does not fit falls
back silently to the step-wise kernels.  Here each case forces a plan with the host switches of DESIGN §7
(LVSR_DEC_CS, LVSR_DEC_LAYOUT, LVSR_DEC_HANDLER, LVSR_ATT_CS), asserts through SpeechRecognizer.decoder_plan() that
this plan ran, and compares every output with O.cost_matrix (content_oracle for content attention):

  * weights: relative error per element wherever the oracle weight is >= 1e-30, < 1e-29 below that, exactly 0
    where the oracle's is 0 (outside the window, masked positions, rows without a valid position);
  * energies: absolute error per element over the tensor's largest magnitude; exactly 0 outside the window;
  * weight sums: within WSUM_TOL of 1 for rows with a valid position, exactly 0 for the others;
  * costs, states, weighted averages: |got - want| <= tol * (|want| + FLOOR * max|want|) per element.

The oracle runs on the float32-rounded inputs and parameters the GPU sees, so the errors measured are the kernels'
own.  The bounds in TOL sit 4-13x above the largest error measured for each quantity over every case of this file on
an H100 80GB HBM3 (700 W power limit); none is looser than 1e-4, the project's gate.  The GRU states and weighted
averages carry absolute errors of about 1e-6 of their scale, so their per-element floor is 0.1 of the scale.  The
file runs in about 20 s on that GPU.

The cases here use E = 256 (BiGRU(128)), where the gate product's K = E + C = 512 is reached as C = 256.  The encoder
gives every E that is a multiple of 128 from 128 to 1024; the other encoded widths, among them E + C = 512 as 384 + 128
and 256 as 128 + 128, are covered by test_gpu_encoded_widths.py.
"""
import math

import numpy as np
import pytest

import content_oracle as CO
from helpers import O, check_grads, make_recognizer, package
from helpers import check_energies as _check_energies, check_weights as _check_weights
from helpers import elementwise_err as _elementwise, f32 as _f32

pytestmark = pytest.mark.gpu

# per-quantity bounds; the largest error measured over every case of this file is in the comment
TOL = dict(weights=5e-5,             # 6.8e-6 relative, per element
           energies=2e-5,            # 2.3e-6 of the tensor's largest magnitude
           costs=1e-5,               # 7.8e-7
           logprobs=2e-6,            # 5.0e-7
           states=1e-4,              # 2.1e-5
           weighted_averages=1e-4)   # 2.2e-5
WSUM_TOL = 2e-6                      # 2.0e-7
FLOOR = 0.1                          # costs, states, weighted averages, logprobs: |want| + FLOOR * max|want|

# one BiGRU(128) layer without subsampling: T' = T, so the tests choose T' freely; the oracle gets `attended` directly
ARCH = dict(num_features=40, dims_bidir=[128], subsample=[1], dim_dec=128, dim_matcher=256, conv_n=8,
            conv_num_filters=10, num_phonemes=32, post_merge_dims=[128], maxout_pieces=2)

FULL = dict(type="expanding", initial_begin=0, initial_end=10000, min_speed=0, max_speed=0)
NARROW = dict(type="expanding", initial_begin=0, initial_end=6, min_speed=0.7, max_speed=2.2)
MEDIAN = dict(type="window_around_median", before=5, after=7)
MEAN = dict(type="window_around_mean", before=6, after=6)
PRIORS = dict(full=FULL, narrow=NARROW, median=MEDIAN, mean=MEAN)

_ATT = "/recognizer/generator/att_trans/conv_att"


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _tp(cs, extra=3):
    """Smallest T' with ceil(T'/cs) >= 16 (the planners' rule for cs > 1), plus `extra` so it is not a multiple of cs."""
    return max(16 * cs, 24) + extra


def _params(cfg, seed, content=False, normalizer="softmax"):
    p = (CO if content else O).init_params(cfg, seed=seed, scale=10.0)
    if normalizer != "softmax":
        # energies in [2, 4]: far from relu's kink (an element there has no meaningful relative error) and from the
        # all-zero relu column that is 0/0 in the reference too
        p[_ATT + "/energy_comp/linear.W"] *= 0.05
        p[_ATT + "/energy_comp/linear.b"][:] = 3.0
    return {k: _f32(v) for k, v in p.items()}


def _inputs(cfg, B, Tp, L, seed, lens=None):
    """attended [T',B,E] in (-1, 1) like a GRU output, its mask, labels and a label mask with trailing zeros."""
    rng = np.random.RandomState(seed)
    E = O.dim_encoded(cfg)
    if lens is None:
        lens = rng.randint(int(math.ceil(0.6 * Tp)), Tp + 1, size=B)
        lens[rng.randint(B)] = Tp
    lens = np.asarray(lens)
    att = _f32(rng.uniform(-1, 1, size=(Tp, B, E)))
    attm = (np.arange(Tp)[:, None] < lens[None, :]).astype(np.float64)
    labels = rng.randint(0, cfg["num_phonemes"] - 1, size=(L, B)).astype(np.int64)
    lm = (np.arange(L)[:, None] < rng.randint(max(1, L - 3), L + 1, size=B)[None, :]).astype(np.float64)
    return att, attm, labels, lm


def _set_env(monkeypatch, cs=None, layout=None, compact=False, att_cs=None):
    for k in ("LVSR_DEC_CS", "LVSR_DEC_LAYOUT", "LVSR_DEC_HANDLER", "LVSR_ATT_CS", "LVSR_NO_DEC_SCAN"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("LVSR_DEC_CHECK", "1")       # launch status 0 and no sentinel word left, or the call fails
    if cs is not None:
        monkeypatch.setenv("LVSR_DEC_CS", str(cs))
    if layout is not None:
        monkeypatch.setenv("LVSR_DEC_LAYOUT", layout)
    if compact:
        monkeypatch.setenv("LVSR_DEC_HANDLER", "compact")
    if att_cs is not None:
        monkeypatch.setenv("LVSR_ATT_CS", str(att_cs))


def _make_content(cfg, params):
    pkg = package()
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": cfg["num_features"]}, input_num_chars={}, eos_label=cfg["eos_label"],
        num_phonemes=cfg["num_phonemes"], dim_dec=cfg["dim_dec"], dims_bidir=cfg["dims_bidir"],
        subsample=cfg["subsample"], dim_matcher=cfg["dim_matcher"], post_merge_dims=cfg["post_merge_dims"],
        post_merge_activation=pkg.Maxout(cfg["maxout_pieces"]), attention_type="content", conv_n=None,
        conv_num_filters=cfg["conv_num_filters"], enc_transition=pkg.GatedRecurrent,
        dec_transition=pkg.GatedRecurrent, data_prepend_eos=False)
    rec.set_parameter_values(params)
    return rec


def _assert_plan(plan, cs, layout, kernel, B, what):
    """The report names the plan that was forced; a forced 8-CTA island plan the device cannot hold is skipped."""
    if not plan["ran"]:
        if cs == 8 and layout == "islands":
            pytest.skip("%d 8-CTA clusters are not co-resident on this device (occupancy query: %d)"
                        % (B, plan["max_clusters"]))
        raise AssertionError("%s: the forced plan was declined and the step-wise kernels ran: %s" % (what, plan))
    assert plan["kernel"] == kernel, (what, plan)
    if cs is not None:
        assert plan["cs"] == cs, (what, plan)
        assert plan["tc_cap"] == -(-plan["_Tp"] // cs), (what, plan)
    if layout == "islands":
        assert plan["nisl"] == -(-B // 16) and plan["grid"] == B * plan["cs"] and plan["nrg"] == 1, (what, plan)
    elif layout == "global":
        assert plan["nisl"] == 0 and plan["nrg"] == -(-B // 16) and plan["grid"] >= B * plan["cs"], (what, plan)


def _compare(got, want, content, what):
    got = {k: v.double().cpu().numpy() for k, v in got.items()}
    errs = {}
    _check_weights(got["weights"], want["weights"], errs)
    if content:
        assert not got["energies"].any(), what
    else:
        _check_energies(got["energies"], want["energies"], errs)
    for k in ("costs", "states", "weighted_averages"):
        errs[k] = _elementwise(got[k], want[k])
    print("ERRS", what, " ".join("%s=%.2e" % kv for kv in sorted(errs.items())))
    for k, e in errs.items():
        bound = WSUM_TOL if k.endswith("_sum") else TOL[k]
        assert e <= bound, (what, k, e, bound)
    return got


def _run_cost(monkeypatch, cfg, params, inputs, content=False, cs=None, layout=None, compact=False, kernel=None):
    """Forced plan -> (GPU outputs, plan); the oracle's outputs alongside."""
    torch = _torch()
    att, attm, labels, lm = inputs
    rec = _make_content(cfg, params) if content else make_recognizer(cfg, params)
    _set_env(monkeypatch, cs=cs, layout=layout, compact=compact)
    got = rec.cost_matrix(labels, lm, torch.as_tensor(att, dtype=torch.float32, device="cuda"),
                          torch.as_tensor(attm, dtype=torch.float32, device="cuda"), return_all=True)
    plan = rec.decoder_plan()
    plan["_Tp"] = att.shape[0]
    assert rec.launch_status() == (0, 0)
    want = (CO if content else O).cost_matrix(cfg, params, att, attm, labels, lm, return_all=True)
    return got, want, plan


def _case(monkeypatch, what, cfg, params, inputs, content=False, cs=None, layout=None, compact=False):
    kernel = "dec_content" if content else ("dec_scan<COMPACT>" if compact else "dec_scan")
    got, want, plan = _run_cost(monkeypatch, cfg, params, inputs, content, cs, layout, compact)
    print("PLAN", what, {k: v for k, v in plan.items() if not k.startswith("_")})
    _assert_plan(plan, cs, layout, kernel, inputs[0].shape[1], what)
    _compare(got, want, content, what)
    return plan


# ---- plan matrix -------------------------------------------------------------------------------------------------

# (attention, cs, layout, compact, prior, normaliser): both attention types x cs x layout, the compact handler at every
# cs, logistic and relu at cs >= 2; the priors rotate through the location cases
MATRIX = [
    ("loc", 1, "islands", False, "full", "softmax"),
    ("loc", 1, "global", False, "narrow", "softmax"),
    ("loc", 2, "islands", False, "median", "softmax"),
    ("loc", 2, "global", False, "mean", "softmax"),
    ("loc", 4, "islands", False, "narrow", "softmax"),
    ("loc", 4, "global", False, "full", "softmax"),
    ("loc", 8, "islands", False, "mean", "softmax"),
    ("loc", 8, "global", False, "median", "softmax"),
    ("loc", 1, "global", True, "median", "softmax"),
    ("loc", 2, "islands", True, "full", "softmax"),
    ("loc", 4, "global", True, "mean", "softmax"),
    ("loc", 8, "global", True, "narrow", "softmax"),
    ("loc", 2, "islands", False, "median", "logistic"),
    ("loc", 2, "global", False, "full", "relu"),
    ("loc", 4, "global", False, "mean", "relu"),
    ("loc", 8, "global", False, "narrow", "logistic"),
    ("content", 1, "islands", False, "full", "softmax"),
    ("content", 1, "global", False, "full", "softmax"),
    ("content", 2, "islands", False, "full", "softmax"),
    ("content", 2, "global", False, "full", "softmax"),
    ("content", 4, "islands", False, "full", "softmax"),
    ("content", 4, "global", False, "full", "softmax"),
    ("content", 8, "islands", False, "full", "softmax"),
    ("content", 8, "global", False, "full", "softmax"),
]


@pytest.mark.parametrize("att,cs,layout,compact,prior,normalizer", MATRIX,
                         ids=["-".join(map(str, c[:3])) + ("-compact" if c[3] else "") + "-%s-%s" % c[4:]
                              for c in MATRIX])
def test_plan_matrix_matches_oracle(att, cs, layout, compact, prior, normalizer, monkeypatch):
    content = att == "content"
    B = 16 if layout == "islands" else 6
    if content:
        cfg = CO.make_config(**ARCH)
    else:
        cfg = O.make_config(prior=PRIORS[prior], energy_normalizer=normalizer, **ARCH)
    params = _params(cfg, seed=cs + 7, content=content, normalizer=normalizer)
    inputs = _inputs(cfg, B, _tp(cs), 8, seed=100 + cs)
    plan = _case(monkeypatch, "matrix", cfg, params, inputs, content, cs, layout, compact)
    if compact:
        assert plan["wh_rows"] == cfg["conv_num_filters"]
    elif not content:
        assert plan["wh_rows"] == 16


def test_red_alias_plan_matches_oracle(monkeypatch):
    """16 rows x T' = 400 at cs 1: 416-position chunks, so the dense tiles' cross-warp scratch lives in the
    attention's reduction scratch."""
    cfg = O.make_config(prior=dict(type="window_around_median", before=20, after=24), **ARCH)
    params = _params(cfg, seed=3)
    plan = _case(monkeypatch, "red_alias", cfg, params, _inputs(cfg, 16, 400, 6, seed=4), cs=1, layout="islands")
    assert plan["red_alias"] == 1


# ---- ragged islands ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B,prior", [(37, "median"), (37, "full"), (33, "mean")])
def test_ragged_islands_match_oracle(B, prior, monkeypatch):
    """37 rows = islands of 13 + 12 + 12, 33 rows = three islands of 11 (not 16): cs 2, T' = 40."""
    cfg = O.make_config(prior=PRIORS[prior], **ARCH)
    params = _params(cfg, seed=B)
    plan = _case(monkeypatch, "ragged", cfg, params, _inputs(cfg, B, 40, 7, seed=B), cs=2, layout="islands")
    assert plan["nisl"] == 3 and plan["ncg"] == (B // 3) * 2


# ---- window and chunk edges at every cs --------------------------------------------------------------------------

@pytest.mark.parametrize("cs", [1, 2, 4, 8])
@pytest.mark.parametrize("edge", ["narrow_window", "short_utterances", "window_reaches_end", "median_tie"])
def test_window_edges_match_oracle(edge, cs, monkeypatch):
    Tp, B, L, lens, params_fix = _tp(cs), 6, 8, None, None
    if edge == "narrow_window":
        # [0, 6) at the first step: at cs 8 the chunk is one position and ranks 6, 7 own none
        prior = dict(type="expanding", initial_begin=0, initial_end=6, min_speed=0.5, max_speed=1.0)
    elif edge == "short_utterances":
        # rows of 1-3 encoded frames: the window [4, ...) holds no valid position of theirs (anyone = 0: zero weights)
        prior = dict(type="expanding", initial_begin=4, initial_end=20, min_speed=1.0, max_speed=3.0)
        lens = [1, 2, 3, Tp, Tp - 5, 3]
    elif edge == "window_reaches_end":
        prior = dict(type="expanding", initial_begin=0, initial_end=6, min_speed=1.0, max_speed=Tp / 3.0)
    else:
        # energies 0: uniform weights over 32 positions, every partial sum exact in fp32 and float64, and half of the
        # mass ends exactly on a rank boundary at every cs > 1 (positions 16 = 2 x 8 = 4 x 4): the median owner rule
        # and the crossing index (15, reported as 14) decide the next step's window.  L = 2: from step 1 on the
        # window holds 46 positions and an exact half is no longer representable.
        prior = dict(type="window_around_median", before=16, after=32)
        Tp = max(Tp, 50)
        lens, L = [Tp] * B, 2
        params_fix = {_ATT + "/energy_comp/linear.W": 0.0}
    cfg = O.make_config(prior=prior, **ARCH)
    params = _params(cfg, seed=11 * cs)
    for k, v in (params_fix or {}).items():
        params[k] = params[k] * v
    inputs = _inputs(cfg, B, Tp, L, seed=cs, lens=lens)
    _case(monkeypatch, edge, cfg, params, inputs, cs=cs, layout="global")
    if edge == "median_tie":
        want = O.cost_matrix(cfg, params, *inputs, return_all=True)
        assert np.all((want["weights"][1] > 0).sum(-1) == 46)         # the step after the tie: positions 0..45


# ---- dense shapes ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("layout,cs,B", [("islands", 2, 16), ("global", 1, 6)])
def test_gate_product_k512_matches_oracle(layout, cs, B, monkeypatch):
    """E + C = 512 (BiGRU(128) encoder, dim_dec 256): 16 k-values per lane in the gate tile (kper = 16)."""
    cfg = O.make_config(prior=MEDIAN, **dict(ARCH, dim_dec=256, post_merge_dims=[256]))
    params = _params(cfg, seed=5)
    plan = _case(monkeypatch, "k512", cfg, params, _inputs(cfg, B, _tp(cs), 6, seed=5), cs=cs, layout=layout)
    # 256 units over the column groups, 8 per tile: the gate tile has 3 x 8 columns
    assert plan["nc2"] == 8 and plan["nc1"] == 24 and plan["ncg"] >= 32


# ---- training through a forced plan ------------------------------------------------------------------------------

@pytest.mark.parametrize("what,B,env", [("ragged_islands_cs2", 37, dict(LVSR_DEC_CS="2", LVSR_DEC_LAYOUT="islands")),
                                        ("compact_handler", 6, dict(LVSR_DEC_HANDLER="compact"))])
def test_gradients_through_forced_plan(what, B, env, monkeypatch):
    """The backward pass consumes the forward's alignments, previous states and contexts (W_all / S_prev / CTX)."""
    _torch()
    _set_env(monkeypatch)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    cfg = O.make_config(prior=MEDIAN, **ARCH)
    params = O.init_params(cfg, seed=7, scale=10.0)
    batch = O.synthetic_batch(cfg, B=B, T=40, seed=12)
    _, rec = check_grads(cfg, params, batch)
    plan = rec.decoder_plan()
    assert plan["ran"], plan
    if what == "compact_handler":
        assert plan["kernel"] == "dec_scan<COMPACT>" and plan["wh_rows"] == cfg["conv_num_filters"], plan
    else:
        assert plan["kernel"] == "dec_scan" and plan["cs"] == 2 and plan["nisl"] == 3, plan


# ---- the attention step kernel -----------------------------------------------------------------------------------

@pytest.mark.parametrize("prior", list(PRIORS))
@pytest.mark.parametrize("cs", [1, 2, 4, 8])
def test_step_kernel_matches_oracle(cs, prior, monkeypatch):
    """logprobs_computer / next_state_computer for several steps at a forced attention-step cluster size."""
    torch = _torch()
    cfg = O.make_config(prior=PRIORS[prior], **ARCH)
    params = _params(cfg, seed=21 + cs)
    Tp, R = _tp(cs), 3
    att, attm, _, _ = _inputs(cfg, R, Tp, 1, seed=cs, lens=[Tp, Tp - 4, Tp - 9])
    rec = make_recognizer(cfg, params)
    _set_env(monkeypatch, att_cs=cs)
    ctx = dict(attended=torch.as_tensor(att, dtype=torch.float32, device="cuda"),
               attended_mask=torch.as_tensor(attm, dtype=torch.float32, device="cuda"))
    st_o = O.initial_states(cfg, params, R, att)
    st_g = rec._initial_states(Tp, R)
    for step in range(6):
        lp_o = O.logprobs_computer(cfg, params, att, attm, st_o)
        lp_g = rec._logprobs(ctx, st_g).double().cpu().numpy()
        assert rec.decoder_plan()["att_cs"] == cs
        errs = dict(logprobs=_elementwise(lp_g, lp_o))
        y = lp_o.argmin(axis=1)
        st_o = O.next_state_computer(cfg, params, att, attm, st_o, y)
        st_g = rec._next_states(ctx, st_g, y)
        g = {k: v.double().cpu().numpy() for k, v in st_g.items()}
        _check_weights(g["weights"], st_o["weights"], errs)
        _check_energies(g["energies"], st_o["energies"], errs)
        errs["states"] = _elementwise(g["states"], st_o["states"])
        errs["weighted_averages"] = _elementwise(g["weighted_averages"], st_o["weighted_averages"])
        print("ERRS step", cs, prior, step, " ".join("%s=%.2e" % kv for kv in sorted(errs.items())))
        for k, e in errs.items():
            assert e <= (WSUM_TOL if k.endswith("_sum") else TOL[k]), (step, k, e)
        assert np.array_equal(g["step"], st_o["step"])


def test_beam_search_at_cs8_gives_the_oracle_tokens(monkeypatch):
    _torch()
    cfg = O.make_config(max_decoded_length_scale=1.0, **ARCH)
    params = O.init_params(cfg, seed=17, scale=10.0)
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.W"] *= 40
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.b"][cfg["eos_label"]] = 24.0
    rec = make_recognizer(cfg, params)
    rec.init_beam_search(4)
    _set_env(monkeypatch, att_cs=8)
    x = np.random.RandomState(3).normal(size=(_tp(8), cfg["num_features"]))
    want_out, want_costs = O.beam_search(cfg, params, x, 4, stop_on="optimistic_future_cost", char_discount=0.1)
    got_out, got_costs = rec.beam_search({"recordings": x}, stop_on="optimistic_future_cost", char_discount=0.1)
    assert rec.decoder_plan()["att_cs"] == 8
    assert got_out == want_out
    assert np.allclose(got_costs, want_costs, rtol=1e-4, atol=1e-4)


# ---- the switches themselves -------------------------------------------------------------------------------------

def test_unfit_forced_plans_are_declined(monkeypatch):
    """A forced plan that breaks a planner rule never launches: the step-wise kernels run and the report says so."""
    torch = _torch()
    cfg = O.make_config(prior=MEAN, **ARCH)
    params = _params(cfg, seed=2)
    att, attm, labels, lm = _inputs(cfg, 6, 40, 5, seed=2)
    want = O.cost_matrix(cfg, params, att, attm, labels, lm, return_all=True)
    rec = make_recognizer(cfg, params)
    for forced in (dict(cs=4),                    # ceil(40 / 4) = 10 < 16
                   dict(layout="islands")):       # 6 rows < one 16-row island
        _set_env(monkeypatch, **forced)
        got = rec.cost_matrix(labels, lm, torch.as_tensor(att, dtype=torch.float32, device="cuda"),
                              torch.as_tensor(attm, dtype=torch.float32, device="cuda"), return_all=True)
        plan = rec.decoder_plan()
        assert not plan["ran"] and plan["kernel"] == "stepwise" and plan["cs"] == 0, (forced, plan)
        assert plan["att_cs"] >= 1, plan                # the step-wise fallback ran the attention step kernel
        _compare(got, want, False, "declined %s" % forced)
    _set_env(monkeypatch, att_cs=8)                     # ceil(40 / 8) = 5 < 16: the planner's own choice runs
    rec._logprobs(dict(attended=torch.as_tensor(att, dtype=torch.float32, device="cuda"),
                       attended_mask=torch.as_tensor(attm, dtype=torch.float32, device="cuda")),
                  rec._initial_states(40, 6))
    assert rec.decoder_plan()["att_cs"] in (1, 2)
    monkeypatch.setenv("LVSR_DEC_CS", "3")
    with pytest.raises(RuntimeError, match="LVSR_DEC_CS"):
        rec.cost_matrix(labels, lm, torch.as_tensor(att, dtype=torch.float32, device="cuda"),
                        torch.as_tensor(attm, dtype=torch.float32, device="cuda"))
