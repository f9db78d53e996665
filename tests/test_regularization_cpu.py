"""Dropout, weight noise and the alignment penalty (regularization.dropout / noise / penalty_coof, lvsr/main.py:400-417)
on the host: Blocks' test_apply_dropout / test_apply_noise restated on the oracle (tests/regularization_oracle.py), the
noise subjects by name, the oracle's gradient at the regularised point, the penalty against the validation statistic,
its hand-written gradient against autograd and finite differences and a tie, GradientDescent's regularization argument
and compat's train handing config['regularization'] through (GPU calls replaced by recording fakes)."""
import logging
import os
import sys

import numpy as np
import pytest

import bottom_oracle as BO
import content_oracle as CO
import regularization_oracle as RO
import training_loop_oracle as TLO
from compat_helpers import COMPAT, write_experiment
from helpers import O, package
from oracle import lvsr_oracle_grad as G

TINY = dict(num_features=6, dims_bidir=[8], subsample=[1], dim_dec=8, dim_matcher=8, conv_n=2, conv_num_filters=2,
            num_phonemes=5, post_merge_dims=[8], maxout_pieces=2, dim_output_embedding=4)


def test_apply_dropout_multiplies_by_mask_over_keep_probability():
    """B/tests/graph/test_graph.py test_apply_dropout: x * mask / (1 - p) with p = 0.5."""
    x = np.arange(12, dtype=np.float64).reshape(2, 3, 2) - 5.0
    mask = (np.arange(12).reshape(2, 3, 2) % 3 != 0).astype(np.float64)
    out = RO.dropout(x, mask)
    assert np.array_equal(out, np.where(mask > 0, 2.0 * x, 0.0))
    assert set(np.unique(RO.dropout(np.ones(100), mask.reshape(-1).repeat(9)[:100]))) <= {0.0, 2.0}


def test_apply_noise_adds_level_times_eps_to_the_subjects_only():
    """B/tests/graph/test_graph.py test_apply_noise: p + N(0, level^2) on the subjects, the others unchanged."""
    cfg = O.make_config(**TINY)
    params = O.init_params(cfg, seed=3)
    rng = np.random.RandomState(0)
    eps = {k: rng.normal(size=v.shape) for k, v in params.items()}
    out = RO.noisy(params, eps, 0.25)
    for k, v in params.items():
        want = v + 0.25 * eps[k] if RO.is_noise_subject(k) else v
        assert np.array_equal(out[k], want), k
    big = {"w": np.zeros(200000)}
    d = RO.noisy(big, {"w": rng.normal(size=200000)}, 0.3)["w"]
    assert abs(d.mean()) < 5 * 0.3 / np.sqrt(d.size) and abs(d.std() - 0.3) < 5 * 0.3 / np.sqrt(2 * d.size)


WSJ_JAN_NEW = dict(num_features=123, dims_bidir=[250, 250, 250, 250], subsample=[1, 1, 2, 2], dim_dec=250,
                   dim_matcher=250, conv_n=100, conv_num_filters=10, num_phonemes=44, post_merge_dims=[250])


@pytest.mark.parametrize("name,cfg", [
    ("wsj_jan_new", O.make_config(**WSJ_JAN_NEW)),
    ("nips_baseline_content", CO.make_config(**WSJ_JAN_NEW)),
    ("logistic", O.make_config(**dict(WSJ_JAN_NEW, energy_normalizer="logistic"))),
    ("bottom", BO.make_config(O.make_config(**WSJ_JAN_NEW), [256], "relu")),
], ids=lambda v: v if isinstance(v, str) else "")
def test_noise_subjects_are_every_parameter_outside_the_attention(name, cfg):
    shapes = (BO.param_shapes(cfg) if cfg.get("bottom") else
              CO.param_shapes(cfg) if cfg.get("attention_type") == "content" else O.param_shapes(cfg))
    excluded = [k for k in shapes if not RO.is_noise_subject(k)]
    subjects = [k for k in shapes if RO.is_noise_subject(k)]
    base = "/recognizer/generator/att_trans/" + ("cont_att" if name.startswith("nips") else "conv_att")
    assert excluded and all(k.startswith(base + "/") for k in excluded)
    leaves = {k[len(base):] for k in excluded}
    assert "/state_trans/transform_states.W" in leaves and "/preprocess.W" in leaves and "/preprocess.b" in leaves
    assert "/energy_comp/linear.W" in leaves
    if name == "logistic":
        assert "/energy_comp/linear.b" in leaves
    if not name.startswith("nips"):
        assert {"/handler.W", "/conv1d.filters"} <= leaves
    for part in ("/recognizer/encoder/bidir0/forward/fork/fork_inputs.W", "/recognizer/generator/att_trans/transition.state_to_gates",
                 "/recognizer/generator/att_trans/distribute/fork_inputs.W", "/recognizer/generator/fork/fork_inputs.W",
                 "/recognizer/generator/readout/post_merge/mlp/linear_0.W",
                 "/recognizer/generator/readout/lookupfeedback/lookuptable.W"):
        assert part in subjects, part
    if name == "bottom":
        assert BO.linear_name(0) + ".W" in subjects and BO.linear_name(0) + ".b" in subjects


def test_oracle_regularised_gradient_is_the_gradient_at_the_regularised_point():
    """Dropout on the recordings is the plain oracle on x * mult; weight noise the plain oracle at p + level eps with
    the attention's parameters clean; with a bottom MLP the multiplier sits between the bottom and the encoder."""
    cfg = O.make_config(**TINY)
    params = O.init_params(cfg, seed=4, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=2, T=7, seed=5)
    mult = 2.0 * (np.random.RandomState(1).rand(*x.shape) < 0.5)
    c0, g0 = RO.cost_and_grads(cfg, params, x, m, labels, lm, mult=mult)
    c1, g1 = G.cost_and_grads(cfg, params, x * mult, m, labels, lm)
    assert c0 == pytest.approx(c1, rel=1e-12)
    for k in g1:
        np.testing.assert_allclose(g0[k], g1[k], rtol=1e-10, atol=1e-14)
    eps = {k: np.random.RandomState(2).normal(size=v.shape) for k, v in params.items()}
    c0, g0 = RO.cost_and_grads(cfg, params, x, m, labels, lm, eps=eps, level=0.05)
    c1, g1 = G.cost_and_grads(cfg, RO.noisy(params, eps, 0.05), x, m, labels, lm)
    assert c0 == pytest.approx(c1, rel=1e-12)
    for k in g1:
        np.testing.assert_allclose(g0[k], g1[k], rtol=1e-10, atol=1e-14)
    bcfg = BO.make_config(cfg, [5], "tanh")
    bparams = BO.init_params(bcfg, seed=6, scale=10.0)
    bmult = 2.0 * (np.random.RandomState(3).rand(x.shape[0], x.shape[1], 5) < 0.5)
    c0, g0 = RO.cost_and_grads(bcfg, bparams, x, m, labels, lm, mult=bmult)
    c1, _ = BO.cost_and_grads(bcfg, bparams, x, m, labels, lm)
    assert c0 != pytest.approx(c1)
    # finite difference through the dropped bottom: d cost / d linear_0.b[0]
    k, h = BO.linear_name(0) + ".b", 1e-6
    up, down = dict(bparams), dict(bparams)
    up[k] = bparams[k] + np.eye(5)[0] * h
    down[k] = bparams[k] - np.eye(5)[0] * h
    fd = (RO.cost_and_grads(bcfg, up, x, m, labels, lm, mult=bmult)[0] -
          RO.cost_and_grads(bcfg, down, x, m, labels, lm, mult=bmult)[0]) / (2 * h)
    assert g0[k][0] == pytest.approx(fd, rel=1e-5, abs=1e-9)


def test_penalty_equals_the_validation_statistic_and_its_gradient_autograd_and_finite_differences():
    """The oracle's weights_penalty is training_loop_oracle's validation statistic; penalty_grad is autograd of the
    torch form (max(., 0) with the [x >= 0] gradient) and, away from ties, central finite differences."""
    import torch
    rng = np.random.RandomState(7)
    L, B, T = 5, 3, 9
    w = rng.rand(L, B, T) ** 3          # unnormalised rows: the cumulative sums end apart too
    m = (np.arange(L)[:, None] < np.array([5, 3, 4])[None, :]).astype(np.float64)
    assert RO.penalty(w, m) == pytest.approx(TLO.alignment_stats(w, m)[1], rel=1e-12)
    assert RO.penalty(w) == pytest.approx(TLO.alignment_stats(w)[1], rel=1e-12)
    g = RO.penalty_grad(w, m)
    wt = torch.tensor(w, requires_grad=True)
    auto = torch.autograd.grad(RO.penalty(wt, torch.tensor(m)), wt)[0].numpy()
    np.testing.assert_allclose(g, auto, rtol=0, atol=1e-12)
    c = np.cumsum(w, axis=2)
    assert np.abs(c[1:] - c[:-1]).min() > 1e-6          # away from ties
    h = 1e-8
    for idx in [(0, 0, 0), (2, 1, 4), (4, 0, 8), (3, 2, 2), (1, 2, 6)]:
        up, down = w.copy(), w.copy()
        up[idx] += h
        down[idx] -= h
        fd = (RO.penalty(up, m) - RO.penalty(down, m)) / (2 * h)
        assert g[idx] == pytest.approx(fd, abs=1e-6), idx


def test_penalty_gradient_counts_a_tie_as_increasing():
    """Two rows both exactly 0 before their windows tie at every early frame: Theano's maximum gives that tie the
    gradient 1, where a clamp / torch.maximum convention would give 0 or 1/2."""
    w = np.zeros((2, 1, 4))
    w[0, 0] = [0.0, 0.0, 1.0, 0.0]
    w[1, 0] = [0.0, 0.0, 0.0, 1.0]
    # c_0 = [0, 0, 1, 1], c_1 = [0, 0, 0, 1]: ties at t = 0, 1, 3; c_1 < c_0 at t = 2
    g = RO.penalty_grad(w)
    assert np.array_equal(g[1, 0], [3.0, 2.0, 1.0, 1.0])
    assert np.array_equal(g[0, 0], [-3.0, -2.0, -1.0, -1.0])
    strict = np.array([0.0, 0.0, 0.0, 0.0])          # what [c_1 > c_0] would give row 1
    assert not np.array_equal(g[1, 0], strict)
    import torch
    wt = torch.tensor(w, requires_grad=True)
    assert np.array_equal(torch.autograd.grad(RO.penalty(wt), wt)[0].numpy(), g)


def test_oracle_penalty_term_is_coof_times_the_penalty_over_b():
    """cost_and_grads with coof: the gradient is the task gradient plus coof / B times the penalty's, the cost stays
    the task cost."""
    cfg = O.make_config(**TINY)
    params = O.init_params(cfg, seed=4, scale=10.0)
    batch = O.synthetic_batch(cfg, B=2, T=16, seed=5)
    c0, g0, pen, w = RO.cost_and_grads(cfg, params, *batch, return_penalty=True)
    c1, g1 = RO.cost_and_grads(cfg, params, *batch, coof=0.5)
    assert c0 == c1 and pen == pytest.approx(RO.penalty(w, batch[3]), rel=1e-12) and pen > 0
    k = "/recognizer/generator/att_trans/conv_att/energy_comp/linear.W"
    assert np.abs(g1[k] - g0[k]).max() > 1e-6
    h = 1e-6
    up, down = dict(params), dict(params)
    up[k] = params[k] + h * np.eye(params[k].shape[0], 1)
    down[k] = params[k] - h * np.eye(params[k].shape[0], 1)
    fd = sum(s * (RO.cost_and_grads(cfg, q, *batch)[0] + 0.5 * RO.cost_and_grads(cfg, q, *batch, return_penalty=True)[2]
                  / 2) for s, q in ((1, up), (-1, down))) / (2 * h)
    assert g1[k][0, 0] == pytest.approx(fd, rel=1e-4, abs=1e-8)


class _Rec(object):
    lm = None


def test_gradient_descent_checks_and_maps_the_regularization_argument(caplog):
    pkg = package()
    gd = pkg.GradientDescent
    assert gd(recognizer=_Rec()).regularization is None
    assert gd(recognizer=_Rec(), regularization=dict(dropout=False, noise=0.0, penalty_coof=0.0)).regularization is None
    assert gd(recognizer=_Rec(), regularization=dict(dropout=True)).regularization == \
        dict(dropout=True, noise=0.0, penalty_coof=0.0, seed=1)
    assert gd(recognizer=_Rec(), regularization=dict(noise=0.075, seed=0)).regularization == \
        dict(dropout=False, noise=0.075, penalty_coof=0.0, seed=1)
    assert gd(recognizer=_Rec(), regularization=dict(penalty_coof=0.5)).regularization == \
        dict(dropout=False, noise=0.0, penalty_coof=0.5, seed=1)
    assert gd(recognizer=_Rec(), regularization=dict(noise=0.1, seed=9)).regularization["seed"] == 9
    with pytest.raises(TypeError):
        gd(recognizer=_Rec(), regularization=dict(dropout=True, weight_noise=0.1))
    with pytest.raises(TypeError):
        gd(recognizer=_Rec(), regularization=dict(dropout=1))
    with pytest.raises(ValueError):
        gd(recognizer=_Rec(), regularization=dict(noise=-0.1))
    with pytest.raises(ValueError):
        gd(recognizer=_Rec(), regularization=dict(penalty_coof=-1.0))
    # lvsr/main.py:402-408 builds the noisy graph from the graph without dropout: with noise, dropout is dropped
    with caplog.at_level(logging.WARNING):
        both = gd(recognizer=_Rec(), regularization=dict(dropout=True, noise=0.075, penalty_coof=0.5))
    assert both.regularization == dict(dropout=False, noise=0.075, penalty_coof=0.5, seed=1)
    assert "dropout has no effect with noise" in caplog.text
    caplog.clear()
    # under adaptive noise the reference trains on the clean graph: the three are logged and dropped
    an = dict(num_examples=10)
    with caplog.at_level(logging.ERROR):
        algo = gd(recognizer=_Rec(), adaptive_noise=an, regularization=dict(dropout=True, noise=0.1, penalty_coof=1.0))
    assert algo.regularization is None and algo.adaptive_noise is not None
    assert "probably stupid" in caplog.text and "no effect under adaptive noise" in caplog.text
    caplog.clear()
    with caplog.at_level(logging.ERROR):
        gd(recognizer=_Rec(), adaptive_noise=an, regularization=dict(dropout=True))
    assert "probably stupid" not in caplog.text and "no effect under adaptive noise" in caplog.text


class _Dist(object):
    def __init__(self, rank):
        self.rank = rank

    def get_rank(self):
        return self.rank


def test_data_parallel_dropout_offset_and_the_unequal_shards_refusal():
    pkg = package()
    batch = dict(recordings=np.zeros((5, 3, 4), np.float32))
    algo = pkg.GradientDescent(recognizer=_Rec(), regularization=dict(dropout=True))
    assert algo._utterance_offset(_Dist(2), batch) == 6
    algo.equal_shards = False
    with pytest.raises(NotImplementedError, match="equal shards"):
        algo._utterance_offset(_Dist(1), batch)
    plain = pkg.GradientDescent(recognizer=_Rec(), regularization=dict(noise=0.1))
    plain.equal_shards = False
    assert plain._utterance_offset(_Dist(1), batch) == 0        # weight noise is keyed by parameter element only


REG_YAML = """
parent: {base}
training:
    num_batches: 1
regularization:
{reg}
"""


@pytest.mark.parametrize("reg,want,logged", [
    ("    dropout: true\n    noise: 0.075", dict(dropout=True, noise=0.075), ["apply dropout", "apply noise"]),
    ("    dropout: true\n    penalty_coof: 0.5", dict(dropout=True, penalty_coof=0.5), ["apply dropout"]),
    ("    dropout: false\n    max_norm: 1.0", None, []),
])
def test_compat_train_hands_the_regularization_through(tmp_path, monkeypatch, caplog, reg, want, logged):
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as LC
    import lvsr.main as M
    exp = write_experiment(tmp_path)
    path = os.path.join(str(tmp_path), "reg.yaml")
    with open(path, "w") as f:
        f.write(REG_YAML.format(base=exp["base"], reg=reg))
    cfg = LC.Configuration(path, "$LVSR/lvsr/configs/schema.yaml", [])
    made = []

    class Stop(Exception):
        pass

    class FakeGD(object):
        def __init__(self, recognizer, step_rule, decay, adaptive_noise, **kwargs):
            made.append(kwargs)
            raise Stop()

    monkeypatch.setattr(M, "create_model", lambda config, data, load_path=None, test_tag=False: _Rec())
    monkeypatch.setattr(M.pkg, "GradientDescent", FakeGD)
    with caplog.at_level(logging.INFO), pytest.raises(Stop):
        M.train(cfg, os.path.join(str(tmp_path), "run.tar"))
    assert made == [{} if want is None else dict(regularization=want)]
    for line in logged:
        assert line in caplog.text
    if not logged:
        assert "apply dropout" not in caplog.text and "apply noise" not in caplog.text
