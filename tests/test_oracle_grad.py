"""Pin the gradient / optimizer oracle (oracle/lvsr_oracle_grad.py):
  * its torch forward mirror equals the numpy oracle (which the reference's frozen sums pin) to 1e-12,
  * autograd gradients agree with central finite differences of the NUMPY oracle's cost,
  * the step rules reproduce the reference's literals
    (libs/blocks/tests/algorithms/test_algorithms.py:80-119,182-249,312-349)."""
from collections import OrderedDict

import numpy as np
import pytest
from numpy.testing import assert_allclose

from oracle import lvsr_oracle as O
from oracle import lvsr_oracle_grad as G

TINY = dict(num_features=5, dims_bidir=[4, 4], subsample=[1, 2], dim_dec=6, dim_matcher=8, conv_n=3,
            conv_num_filters=2, num_phonemes=5, post_merge_dims=[6], maxout_pieces=2)
PRIORS = [None,
          dict(type="expanding", initial_begin=0, initial_end=4, min_speed=0.5, max_speed=1.5),
          dict(type="window_around_median", before=3, after=4),
          dict(type="window_around_mean", before=3, after=3)]


@pytest.mark.parametrize("prior", PRIORS, ids=lambda p: "default" if p is None else p["type"])
@pytest.mark.parametrize("normalizer", ["softmax", "logistic", "relu"])
def test_torch_mirror_equals_numpy_oracle(prior, normalizer):
    cfg = O.make_config(prior=prior, energy_normalizer=normalizer, **TINY)
    params = O.init_params(cfg, seed=4, weights_std=0.3, initial_state_std=0.1)
    if normalizer != "softmax":
        params["/recognizer/generator/att_trans/conv_att/energy_comp/linear.b"][:] = 2.0
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=20, seed=5, label_div=4)
    want = O.recognizer_cost(cfg, params, x, m, labels, lm)
    cost, grads, costs = G.cost_and_grads(cfg, params, x, m, labels, lm, return_costs=True)
    assert_allclose(costs, want, rtol=1e-11, atol=1e-13)
    assert_allclose(cost, O.batch_cost(want), rtol=1e-12)
    assert set(grads) == set(params)
    assert all(np.isfinite(g).all() for g in grads.values())


@pytest.mark.parametrize("prior", [PRIORS[0], PRIORS[2]], ids=["default", "median"])
def test_autograd_matches_finite_differences_of_numpy_oracle(prior):
    cfg = O.make_config(prior=prior, **TINY)
    params = O.init_params(cfg, seed=9, weights_std=0.4, initial_state_std=0.2)
    params["/recognizer/generator/readout/post_merge/bias.b"][:] = np.random.RandomState(0).normal(0, 0.1, 6)
    x, m, labels, lm = O.synthetic_batch(cfg, B=2, T=14, seed=6, label_div=4)
    _, grads = G.cost_and_grads(cfg, params, x, m, labels, lm)
    rng = np.random.RandomState(1)

    def cost_of(p):
        return O.batch_cost(O.recognizer_cost(cfg, p, x, m, labels, lm))
    eps = 1e-6
    for name, value in params.items():
        d = rng.normal(size=value.shape)
        plus = OrderedDict(params); minus = OrderedDict(params)
        plus[name] = value + eps * d
        minus[name] = value - eps * d
        fd = (cost_of(plus) - cost_of(minus)) / (2 * eps)
        an = float((grads[name] * d).sum())
        assert abs(fd - an) <= 1e-6 * max(1.0, abs(an)) + 2e-8, (name, fd, an)


def test_weight_decay_term():
    cfg = O.make_config(**TINY)
    params = O.init_params(cfg, seed=2, weights_std=0.3)
    x, m, labels, lm = O.synthetic_batch(cfg, B=2, T=10, seed=3, label_div=4)
    c0, g0 = G.cost_and_grads(cfg, params, x, m, labels, lm)
    c1, g1 = G.cost_and_grads(cfg, params, x, m, labels, lm, decay=0.01)
    sq = sum((v ** 2).sum() for k, v in params.items() if G.is_weight(k))
    assert_allclose(c1 - c0, 0.01 * sq, rtol=1e-9)       # decay * l2_norm(WEIGHTs)**2, lvsr/main.py:419-421
    for k in params:
        assert_allclose(g1[k] - g0[k], 0.02 * params[k] if G.is_weight(k) else 0 * params[k], atol=1e-12)


# ---- Blocks roles: which parameters decay and max-norm apply to ------------------------------

def _blocks_roles(cfg):
    """The role each recognizer parameter carries in the reference, brick by brick.  VariableFilter(roles=[WEIGHT])
    selects the decay term's and the max-norm's subjects (lvsr/main.py:418-420,493).  Every brick parameter also
    gets the PARAMETER role (B/bricks/base.py:36-44); listed here is the role the brick adds on top, or PARAMETER
    when it adds none."""
    roles = {}
    # GatedRecurrent._allocate: state_to_state WEIGHT (B/bricks/recurrent.py:556), state_to_gates WEIGHT (:560),
    # initial_state INITIAL_STATE (:564)
    # Fork -> Linear: W WEIGHT (B/bricks/simple.py:49), b BIAS (B/bricks/simple.py:54)
    for l in range(len(cfg["dims_bidir"])):
        for d in ("forward", "backward"):
            base = "/recognizer/encoder/bidir%d/%s" % (l, d)
            roles[base + "/gatedrecurrent.state_to_state"] = "WEIGHT"
            roles[base + "/gatedrecurrent.state_to_gates"] = "WEIGHT"
            roles[base + "/gatedrecurrent.initial_state"] = "INITIAL_STATE"
            roles[base + "/fork/fork_inputs.W"] = "WEIGHT"
            roles[base + "/fork/fork_inputs.b"] = "BIAS"
            roles[base + "/fork/fork_gate_inputs.W"] = "WEIGHT"
            roles[base + "/fork/fork_gate_inputs.b"] = "BIAS"
    g, a = "/recognizer/generator", "/recognizer/generator/att_trans"
    if cfg["embed_outputs"]:
        roles[g + "/readout/lookupfeedback/lookuptable.W"] = "WEIGHT"          # LookupTable, B/bricks/lookup.py:42
    if cfg["use_states_for_readout"]:
        roles[g + "/readout/merge/transform_states.W"] = "WEIGHT"              # Merge -> Linear(use_bias=False), simple.py:49
    roles[g + "/readout/merge/transform_weighted_averages.W"] = "WEIGHT"       # simple.py:49
    roles[g + "/readout/post_merge/bias.b"] = "BIAS"                           # Bias, B/bricks/simple.py:95
    roles[g + "/readout/post_merge/mlp/linear_0.W"] = "WEIGHT"                 # simple.py:49
    roles[g + "/readout/post_merge/mlp/linear_0.b"] = "BIAS"                   # simple.py:54
    roles[g + "/fork/fork_inputs.W"] = "WEIGHT"                                # Fork -> Linear, simple.py:49 / :54
    roles[g + "/fork/fork_inputs.b"] = "BIAS"
    roles[g + "/fork/fork_gate_inputs.W"] = "WEIGHT"
    roles[g + "/fork/fork_gate_inputs.b"] = "BIAS"
    roles[a + "/transition.state_to_state"] = "WEIGHT"                         # GatedRecurrent, recurrent.py:556
    roles[a + "/transition.state_to_gates"] = "WEIGHT"                         # recurrent.py:560
    roles[a + "/transition.initial_state"] = "INITIAL_STATE"                   # recurrent.py:564
    roles[a + "/conv_att/state_trans/transform_states.W"] = "WEIGHT"           # Linear(use_bias=False), simple.py:49
    roles[a + "/conv_att/preprocess.W"] = "WEIGHT"                             # Linear, simple.py:49 / :54
    roles[a + "/conv_att/preprocess.b"] = "BIAS"
    roles[a + "/conv_att/energy_comp/linear.W"] = "WEIGHT"                     # MLP -> Linear, simple.py:49
    roles[a + "/conv_att/handler.W"] = "WEIGHT"                                # Linear(use_bias=False), simple.py:49
    roles[a + "/conv_att/conv1d.filters"] = "PARAMETER"                        # Conv1D._allocate adds no role (lvsr/bricks/attention.py:31-33)
    roles[a + "/distribute/fork_inputs.W"] = "WEIGHT"                          # Distribute -> Fork -> Linear(use_bias=False)
    roles[a + "/distribute/fork_gate_inputs.W"] = "WEIGHT"
    return roles


@pytest.mark.parametrize("variant", [{}, dict(embed_outputs=False), dict(use_states_for_readout=False)],
                         ids=["wsj", "one_of_n_feedback", "no_states_for_readout"])
def test_weight_role_table_of_the_wsj_model(variant):
    """G.is_weight is True exactly for the WEIGHT-role parameters of the WSJ model: the conv filters are not among them,
    so neither decay nor max-norm touches them."""
    cfg = O.make_config(num_features=40, dims_bidir=[256] * 4, subsample=[1, 1, 2, 2], dim_dec=256, dim_matcher=512,
                        conv_n=100, conv_num_filters=10, num_phonemes=32, post_merge_dims=[256], maxout_pieces=2,
                        **variant)
    roles = _blocks_roles(cfg)
    names = list(O.param_shapes(cfg))
    assert sorted(names) == sorted(roles)
    wrong = {k: roles[k] for k in names if G.is_weight(k) != (roles[k] == "WEIGHT")}
    assert not wrong, wrong


# ---- step rules: the reference's literals ---------------------------------------------------

def _grad_a(a):
    return 2 * a            # cost = (a ** 2).sum()


def test_momentum_literals():
    a = np.array([3.0, 4.0])
    st = {}
    for want in ([6., 8.], [9., 12.], [10.5, 14.]):            # BasicMomentum(0.5): test_algorithms.py:80-88
        got = G.momentum(OrderedDict(a=_grad_a(a)), st, 1.0, 0.5)["a"]
        assert_allclose(got, want)
    st = {}
    for want in ([0.6, 0.8], [0.9, 1.2], [1.05, 1.4]):          # Momentum(0.1, 0.5): :95-103
        assert_allclose(G.momentum(OrderedDict(a=_grad_a(a)), st, 0.1, 0.5)["a"], want)


def test_adadelta_literals():
    a = np.array([3.0, 4.0])
    st = {}
    for want in (0.00044721, 0.0005164, 0.00056904):           # :110-119
        got = G.adadelta(OrderedDict(a=_grad_a(a)), st, 0.5, 1e-7)["a"]
        assert_allclose(got, [want, want], rtol=1e-5)


def test_step_clipping_literals():
    g = OrderedDict([(0, np.float64(3.0)), (1, np.float64(4.0))])
    c1 = G.step_clipping(g, 4)
    assert_allclose([c1[0], c1[1]], [12 / 5.0, 16 / 5.0])       # :182-193
    c2 = G.step_clipping(g, 5)
    assert_allclose([c2[0], c2[1]], [3.0, 4.0])


def test_variable_clipping_literals():
    assert_allclose(G.variable_clipping(np.array([1., 1]), np.array([3., 2]), 5), [3, 2])          # :200-214
    assert_allclose(G.variable_clipping(np.array([-1., -1, -1]), np.array([[3., 9, 2]]), 5),
                    [[0.78885438, 3.47213595, 0.34164079]], rtol=1e-5)
    p = np.array([[[1.], [-1], [1], [-1]]]); s = np.array([[[1.], [2], [3], [2]]])
    assert_allclose(G.variable_clipping(p, s, 5), s)
    p = np.array([[1., -1, 1, -1], [-1, 1, -1, 1]]); s = np.array([[1., 2, 3, 4], [5, 6, 7, 8]])    # axis=1, :217-226
    assert_allclose(G.variable_clipping(p, s, 10, axis=1),
                    [[1, 2, 3, 4], [3.54858826, 4.79049022, 5.06478435, 6.30668631]], rtol=1e-5)
    p = np.array([[[[1.], [-1]], [[-1], [1]]], [[[-1], [1]], [[2], [-1]]]])
    s = np.array([[[[1.], [2]], [[3], [4]]], [[[5], [6]], [[7], [8]]]])                           # axis=(1,2), :229-245
    assert_allclose(G.variable_clipping(p, s, 10, axis=(1, 2)),
                    [[[[1], [2]], [[3], [4]]], [[[3.6429394], [4.86911616]], [[5.86911616], [5.96440909]]]], rtol=1e-5)
    with pytest.raises(ValueError):
        G.variable_clipping(np.array([1.0]), np.array([1.0]), 10, axis=(1, 2))


def test_remove_not_finite_literals():
    # gradients keyed by "parameter" 1, 2, 3 with those very values as parameters: :312-325
    assert_allclose(G.remove_not_finite(1.0, np.float64(np.nan), 0.1), 0.9)
    assert_allclose(G.remove_not_finite(2.0, np.float64(np.inf), 0.1), 1.8)
    assert_allclose(G.remove_not_finite(3.0, np.float64(0.123), 0.1), 0.123)
    assert_allclose(G.remove_not_finite(1.0, np.float64(np.nan)), 0.0)
    assert_allclose(G.remove_not_finite(2.0, np.float64(np.inf)), 0.0)


def test_composite_chain_of_lvsr_main():
    """lvsr/main.py:480-516 with the WSJ settings (momentum 0 + AdaDelta + max-norm + RemoveNotFinite(0.0))."""
    cfg = O.make_config(**TINY)
    params = O.init_params(cfg, seed=2, weights_std=0.3)
    x, m, labels, lm = O.synthetic_batch(cfg, B=2, T=10, seed=3, label_div=4)
    tc = G.make_train_config(gradient_threshold=0.5, max_norm=0.5, epsilon=1e-6)
    state = {}
    p1, cost1, g1 = G.train_step(cfg, params, state, (x, m, labels, lm), tc)
    assert G.l2_norm(g1.values()) > 0.5                         # so the clipping is active in this test
    for k, v in p1.items():
        if G.is_weight(k):                                     # columns respect the max-norm after the update
            assert (np.sqrt((v ** 2).sum(axis=0)) <= 0.5 + 1e-12).all(), k
    p2, cost2, _ = G.train_step(cfg, p1, state, (x, m, labels, lm), tc)
    assert set(state) == {"velocity", "mean_square_step", "mean_square_delta_x"}
    assert np.isfinite(cost2)
    # a non-finite gradient zeroes that parameter (RemoveNotFinite(0.0)) and leaves the others stepping
    grads = OrderedDict((k, v.copy()) for k, v in g1.items())
    first = next(iter(grads))
    grads[first][...] = np.nan
    steps = G.apply_step_rules(OrderedDict((k, np.asarray(v)) for k, v in params.items()), grads, {}, dict(tc, gradient_threshold=0))
    assert_allclose(params[first] - steps[first], 0.0)
    # burn-in: no update while steps remain (lvsr/algorithms.py:35-43)
    st = {}
    tcb = dict(tc, burn_in_steps=2)
    for i in range(3):
        steps = G.apply_step_rules(params, g1, st, tcb)
        total = sum(np.abs(s).sum() for s in steps.values())
        assert (total == 0) == (i < 2)
