"""The decoder at the encoded widths only a forward-only encoder gives, E = dims[-1] = 64, 192, 320 and 448 (no
bidirectional layer gives an E that is not a multiple of 128), compared with the float64 oracle element by element.

At these widths attention_row splits its partial weighted average into E / 4 column groups and min(8, 512 / (E / 4))
position groups: 8 at E = 64 and 192, 6 at E = 320 (a count no bidirectional width gives) and 4 at E = 448; the
attention backward's loops `for (e = lane * 4; e < E; e += 128)` end within their first pass at E = 64.  The persistent
decoder needs kper_ok(E + C), so every cost here runs the step-wise kernels.  As in test_gpu_encoded_widths.py, each
cost and step case builds a one-layer forward-only encoder of width E and hands `attended` to the decoder directly, so
the oracle (tests/unidirectional_oracle.py, i.e. lvsr_oracle's decoder at E) never runs the encoder:

  * teacher-forced costs under the median and stress window priors and with content attention, B = 6, T' = 40, with
    the attention step's cluster size restated from test_gpu_stepwise_rows.py;
  * LVSR_ATT_CS = 1, 2, 4 and 8 at E = 64 and 320;
  * 72-row greedy steps at E = 64 and 320;
  * gradients at E = 64 and 192 with both attention types (through the encoder, helpers.check_unidirectional_grads).

Bars: test_gpu_attention_plans.py's TOL and WSUM_TOL, test_gpu_encoded_widths.py's STEP_TOL, and check_grads' 1e-4.
Worst errors measured over every case on an H100 80GB HBM3 (700 W power limit): weights 4.9e-6 (bound 5e-5), energies
1.3e-6 (2e-5), weight sums 1.4e-7 (2e-6), costs 3.6e-7 (1e-5), states 1.4e-5 and weighted averages 1.3e-5 (1e-4),
log-probabilities 5.6e-7 (4e-6), gradients 3.1e-6 of a parameter's largest entry (1e-4).  The file runs in about 10 s."""
import numpy as np
import pytest

import unidirectional_oracle as U
from helpers import O, check_unidirectional_grads, f32, make_recognizer
from test_gpu_attention_plans import PRIORS as _PRIORS, _compare, _inputs, _set_env, _tp
from test_gpu_encoded_widths import _greedy
from test_gpu_stepwise_rows import STRESS, _expected_cs

pytestmark = pytest.mark.gpu

PRIORS = dict(_PRIORS, stress=STRESS)
WIDTHS = [64, 192, 320, 448]


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _config(E, prior="median"):
    """A forward-only [E] encoder, C = 128, M = 256, 8 filters of 17 taps; prior None: content attention, "default":
    the default prior."""
    arch = dict(num_features=40, dims_bidir=[E], subsample=[1], dim_dec=128, dim_matcher=256, conv_n=8,
                conv_num_filters=10, num_phonemes=32, post_merge_dims=[128], maxout_pieces=2)
    if prior is None:
        return U.make_config(attention_type="content", **arch)
    if prior == "default":
        return U.make_config(**arch)
    return U.make_config(prior=PRIORS[prior], **arch)


def _params(cfg, seed):
    return {k: f32(v) for k, v in U.init_params(cfg, seed=seed, scale=10.0).items()}


def _cost(monkeypatch, cfg, params, inputs, what, att_cs=None):
    """cost_matrix on `attended` against U.cost_matrix; returns the decoder plan."""
    torch = _torch()
    att, attm, labels, lm = inputs
    rec = make_recognizer(cfg, params, bidir=False)
    _set_env(monkeypatch, att_cs=att_cs)
    got = rec.cost_matrix(labels, lm, torch.as_tensor(att, dtype=torch.float32, device="cuda"),
                          torch.as_tensor(attm, dtype=torch.float32, device="cuda"), return_all=True)
    plan = rec.decoder_plan()
    print("PLAN", what, plan)
    assert rec.launch_status() == (0, 0)
    want = U.cost_matrix(cfg, params, att, attm, labels, lm, return_all=True)
    _compare(got, want, cfg["attention_type"] == "content", what)
    assert rec.dim_encoded == cfg["dims_bidir"][-1]
    return plan


@pytest.mark.parametrize("prior", ["median", "stress", None], ids=["median", "stress", "content"])
@pytest.mark.parametrize("E", WIDTHS)
def test_cost_matrix_matches_oracle(E, prior, monkeypatch):
    """Teacher-forced costs, B = 6, T' = 40, on the step-wise kernels at the planner's attention-step cluster size."""
    B, Tp = 6, 40
    cfg = _config(E, prior)
    params = _params(cfg, seed=E + len(prior or ""))
    inputs = _inputs(U.decoder_config(cfg), B, Tp, 7, seed=E // 64 + 3)
    what = "E=%d %s" % (E, prior or "content")
    plan = _cost(monkeypatch, cfg, params, inputs, what)
    assert not plan["ran"] and plan["kernel"] == "stepwise", (what, plan)
    assert plan["att_cs"] == _expected_cs(B, Tp, prior is not None, M=256, E=E, n=8), (what, plan)


FORCED = [(E, cs) for E in (64, 320) for cs in (1, 2, 4, 8)]


@pytest.mark.parametrize("E,cs", FORCED, ids=["E%d-cs%d" % c for c in FORCED])
def test_forced_attention_step_cluster_sizes(E, cs, monkeypatch):
    """LVSR_ATT_CS = cs at T' = _tp(cs) (ceil(T' / cs) >= 16, not a multiple of cs): attention_row's position groups
    are 8 at E = 64 and 6 at E = 320 (min(8, 512 / (E / 4)))."""
    assert min(8, 512 // (E // 4)) == {64: 8, 320: 6}[E]
    prior = ("median", "stress")[cs.bit_length() % 2]
    cfg = _config(E, prior)
    params = _params(cfg, seed=E + cs)
    inputs = _inputs(U.decoder_config(cfg), 6, _tp(cs), 6, seed=E + 10 * cs)
    plan = _cost(monkeypatch, cfg, params, inputs, "E=%d att_cs %d %s" % (E, cs, prior), att_cs=cs)
    assert not plan["ran"] and plan["kernel"] == "stepwise" and plan["att_cs"] == cs, plan


@pytest.mark.parametrize("E", [64, 320])
def test_greedy_steps_match_oracle(E, monkeypatch):
    """Four greedy steps of 72 rows (more than the persistent kernel's 64) at T' = 40: log-probabilities, weights,
    energies, states and weighted averages against the oracle after every step (test_gpu_encoded_widths._greedy)."""
    cfg = _config(E, "median")
    params = _params(cfg, seed=E + 1)
    dcfg = U.decoder_config(cfg)          # the oracle's view: lvsr_oracle's decoder at E
    Tp = 40
    att, attm, _, _ = _inputs(dcfg, 72, Tp, 1, seed=E)
    rec = make_recognizer(cfg, params, bidir=False)
    cs = _greedy(monkeypatch, dcfg, params, rec, att, attm, 4, "greedy E=%d" % E, dict(M=256, E=E, n=8))
    print("E=%d: attention step cluster size %d" % (E, cs))


GRADS = [(E, attention) for E in (64, 192) for attention in ("content_and_conv", "content")]


@pytest.mark.parametrize("E,attention", GRADS, ids=["E%d-%s" % c for c in GRADS])
def test_gradients_match_oracle(E, attention):
    """Gradients of every parameter through the attention backward (att_bwd_kernel / att_bwd_content_kernel at
    E = 64 and 192) and the forward-only encoder, B = 4, T = 32, at check_grads' bar."""
    _torch()
    cfg = _config(E, "default" if attention == "content_and_conv" else None)
    params = _params(cfg, seed=E + 5)
    x, m, labels, lm = O.synthetic_batch(cfg, B=4, T=32, seed=E + 6)
    rec = check_unidirectional_grads(cfg, params, (f32(x), m, labels, lm))
    plan = rec.decoder_plan()
    print(E, attention, plan, rec.encoder_plan()[0])
    assert not plan["ran"] and rec.encoder_plan()[0]["bwd_cs"] == E // 32 and rec.dim_encoded == E
