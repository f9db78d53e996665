"""Pin the content-only attention oracle (tests/content_oracle.py: attention_type content, SequenceContentAttention
"cont_att"): parameter table, the reference's frozen attention sums through its composite functions, the equivalence
with a zero-handler content_and_conv model, and the torch gradient mirror."""
from collections import OrderedDict

import numpy as np
import pytest
from numpy.testing import assert_allclose

from oracle import lvsr_oracle as O

import content_oracle as CO

CONT = CO.CONT
TR = "/recognizer/generator/att_trans"
TINY = dict(num_features=5, dims_bidir=[4, 4], subsample=[1, 2], dim_dec=6, dim_matcher=8, conv_n=3,
            conv_num_filters=2, num_phonemes=5, post_merge_dims=[6], maxout_pieces=2)


def test_content_param_shapes_in_blocks_order():
    cfg = CO.make_config(**TINY)
    shapes = CO.param_shapes(cfg)
    names = list(shapes)
    C, M, E = 6, 8, 8
    tail = [(TR + "/transition.state_to_state", (C, C)), (TR + "/transition.state_to_gates", (C, 2 * C)),
            (TR + "/transition.initial_state", (C,)),
            (CONT + "/state_trans/transform_states.W", (C, M)), (CONT + "/preprocess.b", (M,)),
            (CONT + "/preprocess.W", (E, M)), (CONT + "/energy_comp/linear.W", (M, 1)),
            (TR + "/distribute/fork_inputs.W", (E, C)), (TR + "/distribute/fork_gate_inputs.W", (E, 2 * C))]
    assert [(n, shapes[n]) for n in names[-len(tail):]] == tail
    assert not any("conv_att" in n or "handler" in n or "conv1d" in n for n in names)
    # everything before the attention is the content_and_conv table's
    conv = list(O.param_shapes(O.make_config(**TINY)))
    assert names[:-len(tail)] == conv[:len(names) - len(tail)]
    # the reference does not pass the normaliser to SequenceContentAttention: no energy bias either way
    assert list(CO.param_shapes(CO.make_config(energy_normalizer="logistic", **TINY))) == names


def _rand(rng, size):
    return rng.uniform(size=size)


def _generate_mask(rng, length, batch_size):
    mask = np.ones((length, batch_size))
    for i in range(batch_size):
        mask[1 + rng.randint(0, length - 1):, i] = 0.0
    return mask


def test_content_attention_freeze_sums_through_take_glimpses():
    """libs/blocks/tests/bricks/test_attention.py:61-135 (SequenceContentAttention inside AttentionRecurrent)
    through CO.initial_glimpses / CO.take_glimpses, the functions the CUDA path is compared with."""
    dim, batch, in_len, att_dim, att_len = 5, 4, 20, 10, 15
    init = np.random.RandomState(1234)
    g = lambda shape: init.normal(0, 0.5, size=shape)
    W_rec = g((dim, dim))
    W_state = g((dim, att_dim))
    W_pre = g((att_dim, att_dim))
    v = g((att_dim, 1))
    W_dist = g((att_dim, dim))

    rng = np.random.RandomState(1234)
    inputs = _rand(rng, (in_len, batch, dim))
    inputs_mask = _generate_mask(rng, in_len, batch)
    attended = _rand(rng, (att_len, batch, att_dim))
    attended_mask = _generate_mask(rng, att_len, batch)

    # a window prior and a non-softmax normaliser are ignored, as SequenceContentAttention takes neither
    cfg = CO.make_config(num_features=3, dims_bidir=[att_dim // 2], dim_dec=dim, dim_matcher=att_dim,
                         num_phonemes=4, attention_type="content", energy_normalizer="logistic",
                         prior=dict(type="window_around_median", before=1, after=1))
    params = {CONT + "/state_trans/transform_states.W": W_state, CONT + "/preprocess.W": W_pre,
              CONT + "/preprocess.b": np.zeros(att_dim), CONT + "/energy_comp/linear.W": v}
    P = CO.preprocess(params, attended)
    assert_allclose(P, attended.dot(W_pre))

    s = np.zeros((batch, dim))
    ctx0, w, e, step = CO.initial_glimpses(cfg, batch, attended)
    assert not ctx0.any() and not w.any() and not e.any()          # B/bricks/attention.py:392-395: zeros
    states, glimpses, weights = [], [], []
    for t in range(in_len):
        ctx, w, e, step = CO.take_glimpses(cfg, params, attended, P, attended_mask, w, step, s)
        assert not e.any()
        s = O.simple_recurrent_step(s, inputs[t] + ctx.dot(W_dist), W_rec, inputs_mask[t],
                                    activation=lambda z: z)
        states.append(s); glimpses.append(ctx); weights.append(w)
    states, glimpses, weights = map(np.stack, (states, glimpses, weights))
    assert np.all(weights * (1 - attended_mask.T) == 0)
    assert_allclose(weights.sum(), in_len * batch, 1e-5)
    assert_allclose(states.sum(), 113.429, rtol=1e-5)
    assert_allclose(glimpses.sum(), 415.901, rtol=1e-5)
    ctx2, _, _, _ = CO.take_glimpses(cfg, params, attended, None, attended_mask, w, step, s)
    ctx1, _, _, _ = CO.take_glimpses(cfg, params, attended, P, attended_mask, w, step, s)
    assert_allclose(ctx1, ctx2, rtol=1e-12)


def test_content_equals_conv_attention_with_zero_handler_and_full_window():
    """A content_and_conv model whose handler is zero, under the default (full-window) prior, computes the same
    costs and weights as the content model with the shared parameters."""
    cfg = CO.make_config(**TINY)
    params = CO.init_params(cfg, seed=4, weights_std=0.3, initial_state_std=0.1)
    ccfg = O.make_config(**TINY)
    cparams = OrderedDict((k.replace("cont_att", "conv_att"), v) for k, v in params.items())
    cparams[O._ATT + "/handler.W"] = np.zeros((2, 8))
    cparams[O._ATT + "/conv1d.filters"] = np.random.RandomState(0).normal(size=(2, 7))
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=20, seed=5, label_div=4)
    a = CO.recognizer_cost(cfg, params, x, m, labels, lm, return_all=True)
    b = O.recognizer_cost(ccfg, cparams, x, m, labels, lm, return_all=True)
    assert_allclose(a["costs"], b["costs"], rtol=1e-12)
    assert_allclose(a["weights"], b["weights"], rtol=1e-12, atol=1e-15)
    assert not a["energies"].any()


def test_content_torch_mirror_equals_numpy_oracle():
    cfg = CO.make_config(**TINY)
    params = CO.init_params(cfg, seed=4, weights_std=0.3, initial_state_std=0.1)
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=20, seed=5, label_div=4)
    want = CO.recognizer_cost(cfg, params, x, m, labels, lm)
    cost, grads, costs = CO.cost_and_grads(cfg, params, x, m, labels, lm, return_costs=True)
    assert_allclose(costs, want, rtol=1e-11, atol=1e-13)
    assert_allclose(cost, O.batch_cost(want), rtol=1e-12)
    assert set(grads) == set(params)
    assert all(np.isfinite(g).all() and np.abs(g).max() > 0 for g in grads.values())


def test_content_autograd_matches_finite_differences_of_numpy_oracle():
    cfg = CO.make_config(**TINY)
    params = CO.init_params(cfg, seed=9, weights_std=0.4, initial_state_std=0.2)
    params["/recognizer/generator/readout/post_merge/bias.b"][:] = np.random.RandomState(0).normal(0, 0.1, 6)
    x, m, labels, lm = O.synthetic_batch(cfg, B=2, T=14, seed=6, label_div=4)
    _, grads = CO.cost_and_grads(cfg, params, x, m, labels, lm)
    rng = np.random.RandomState(1)

    def cost_of(p):
        return O.batch_cost(CO.recognizer_cost(cfg, p, x, m, labels, lm))
    eps = 1e-6
    for name, value in params.items():
        d = rng.normal(size=value.shape)
        plus = OrderedDict(params); minus = OrderedDict(params)
        plus[name] = value + eps * d
        minus[name] = value - eps * d
        fd = (cost_of(plus) - cost_of(minus)) / (2 * eps)
        an = float((grads[name] * d).sum())
        assert abs(fd - an) <= 1e-6 * max(1.0, abs(an)) + 2e-8, (name, fd, an)


def test_content_beam_search_uses_the_content_state_functions():
    """CO.beam_search = the oracle's BeamSearch host logic over the content state functions: the greedy search
    (beam 1, no end-of-line in reach) follows CO.generate_greedy."""
    cfg = CO.make_config(**TINY)
    params = CO.init_params(cfg, seed=3, weights_std=0.5, scale=3.0)
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.b"][cfg["eos_label"]] = -50.0
    x = np.random.RandomState(2).normal(size=(12, 5))
    att, attm = O.encoder(cfg, params, x[:, None, :], None)
    ys, costs, st = CO.generate_greedy(cfg, params, att, attm, 5)
    assert not st["energies"].any() and np.allclose(st["weights"].sum(), 1.0)
    with pytest.raises(O.CandidateNotFoundError):       # end-of-line never chosen: nothing finishes
        CO.beam_search(cfg, params, x, 1, max_length=5)
