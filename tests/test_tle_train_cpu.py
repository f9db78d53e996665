"""Task-loss-estimation training on the host: the float64 gradient oracle of tests/tle_grad_oracle.py against
tests/tle_oracle.py and finite differences, the greedy prediction's mask, and the exploration settings GradientDescent
and compat's train accept or refuse."""
import sys

import numpy as np
import pytest

import tle_grad_oracle as TG
import tle_oracle as TO
from compat_helpers import COMPAT, write_experiment
from helpers import O, SMALL, package

TINY = dict(num_features=6, dims_bidir=[4], subsample=[1], dim_dec=4, dim_matcher=4, conv_n=2, conv_num_filters=2,
            num_phonemes=7, post_merge_dims=[4], maxout_pieces=2)


def _encode(cfg, params, x, m):
    import torch
    from oracle import lvsr_oracle_grad as G
    p = {k: torch.as_tensor(np.asarray(v, dtype=np.float64)) for k, v in params.items()}
    att, am = G._encoder(cfg, p, torch.as_tensor(x), torch.as_tensor(m))
    return p, att, am


def _ragged(cfg, seed, B=3, T=12):
    x, m, labels, lm = O.synthetic_batch(cfg, B=B, T=T, seed=seed)
    return x, m, labels, lm


@pytest.mark.parametrize("name", ["mse_gain", "mse_reward"])
@pytest.mark.parametrize("min_reward", [-1.0, -5.0])
def test_mirror_matches_the_numpy_cost_matrix(name, min_reward):
    """The torch mirror of the loss rows equals tle_oracle.cost_matrix to 1e-12, on ragged label masks, with the labels
    as their own groundtruth and against another groundtruth (a prediction that is not the labels)."""
    import torch
    cfg = O.make_config(**TINY)
    params = O.init_params(cfg, seed=5, scale=3.0)
    x, m, labels, lm = _ragged(cfg, 11)
    p, att, am = _encode(cfg, params, x, m)
    crit = dict(name=name, min_reward=min_reward)
    rng = np.random.RandomState(3)
    prediction = rng.randint(0, cfg["num_phonemes"], size=(labels.shape[0] + 4, labels.shape[1]))
    pmask = TG.prediction_mask(prediction, cfg["eos_label"])
    assert prediction.shape != labels.shape or not np.array_equal(prediction, labels)
    for y, ym, g in ((labels, lm, None), (prediction, pmask, labels)):
        want = TO.cost_matrix(cfg, params, att.numpy(), am.numpy(), y, ym, crit, groundtruth=g)
        got = TG.cost_matrix_torch(cfg, p, att, am, y, torch.as_tensor(ym), crit, groundtruth=g).numpy()
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12 * np.abs(want).max())


@pytest.mark.parametrize("encoder", ["forward_only", "bottom"])
def test_mirror_encoders(encoder):
    """Behind a forward-only encoder and a bottom MLP, the mirror's cost equals tle_oracle.cost_matrix on the numpy
    encoders' output (unidirectional_oracle, bottom_oracle) to 1e-12."""
    import bottom_oracle as BO
    import unidirectional_oracle as U
    if encoder == "forward_only":
        cfg = U.make_config(**TINY)
        params = U.init_params(cfg, seed=5, scale=3.0)
        x, m, labels, lm = _ragged(cfg, 17)
        att, am = U.encoder(cfg, params, x, m)
        dcfg = U.decoder_config(cfg)
    else:
        cfg = BO.make_config(O.make_config(**TINY), [5, 6], activation="tanh")
        params = BO.init_params(cfg, seed=5, scale=3.0)
        x, m, labels, lm = _ragged(cfg, 19)
        att, am = BO.encoder(cfg, params, x, m)
        dcfg = BO.inner(cfg)
    crit = dict(name="mse_reward", min_reward=-1.0)
    want = TO.cost_matrix(dcfg, params, att, am, labels, lm, crit).sum() / labels.shape[1]
    got, _ = TG.cost_and_grads(cfg, params, x, m, labels, lm, crit)
    assert abs(got - want) <= 1e-12 * abs(want), (got, want)


@pytest.mark.parametrize("name", ["mse_gain", "mse_reward"])
@pytest.mark.parametrize("greedy", [False, True])
def test_autograd_matches_finite_differences(name, greedy):
    """The mirror's gradient of every parameter of a tiny model equals central differences of the numpy oracle's
    sum(cost_matrix) / B, for imitative exploration and for a prediction scored against the labels."""
    cfg = O.make_config(**TINY)
    params = O.init_params(cfg, seed=7, scale=3.0)
    x, m, labels, lm = _ragged(cfg, 13, B=2, T=10)
    crit = dict(name=name, min_reward=-1.0)
    if greedy:
        _, att, am = _encode(cfg, params, x, m)
        prediction = TO.generate_greedy(cfg, params, att.numpy(), am.numpy(), labels.shape[0] + TG.EXTRA_STEPS)[0]
        # generate() feeds its picks back without a mask: the oracle's readouts along them pick them again
        assert TG.check_greedy(TG.greedy_readouts(cfg, params, x, m, prediction), prediction, 0.0) == 0
        y, ym, g = prediction, TG.prediction_mask(prediction, cfg["eos_label"]), labels
    else:
        y, ym, g = labels, lm, None
    _, grads = TG.cost_and_grads(cfg, params, x, m, y, ym, crit, groundtruth=g)

    def cost(pp):
        _, att, am = _encode(cfg, pp, x, m)
        return TO.cost_matrix(cfg, pp, att.numpy(), am.numpy(), y, ym, crit, groundtruth=g).sum() / y.shape[1]

    rng = np.random.RandomState(0)
    eps = 1e-6
    for k, v in params.items():
        v = np.asarray(v, dtype=np.float64)
        for idx in {tuple(rng.randint(0, s) for s in v.shape) for _ in range(3)}:
            hi, lo = dict(params), dict(params)
            hi[k], lo[k] = v.copy(), v.copy()
            hi[k][idx] += eps
            lo[k][idx] -= eps
            fd = (cost(hi) - cost(lo)) / (2 * eps)
            assert abs(grads[k][idx] - fd) <= 1e-5 * max(1.0, abs(fd)), (k, idx, grads[k][idx], fd)


def _add_exploration_mask(prediction, eos):
    """lvsr/main.py:252-258 restated step by step: m[0] = 1, m[t] = 1 iff no eos in prediction[0 .. t-1]."""
    n, B = prediction.shape
    m = np.zeros((n, B))
    for b in range(B):
        for t in range(n):
            m[t, b] = 1.0 if t == 0 or eos not in list(prediction[:t, b]) else 0.0
    return m


def test_prediction_mask():
    eos = 3
    cols = [
        [3, 1, 2, 0, 1, 2],          # eos at step 0
        [1, 2, 3, 0, 1, 2],          # eos mid-way
        [1, 3, 2, 3, 0, 3],          # several eos
        [1, 2, 0, 1, 2, 0],          # none in all steps
    ]
    prediction = np.array(cols).T
    want = _add_exploration_mask(prediction, eos)
    np.testing.assert_array_equal(TG.prediction_mask(prediction, eos), want)
    np.testing.assert_array_equal(want[:, 0], [1, 0, 0, 0, 0, 0])
    np.testing.assert_array_equal(want[:, 1], [1, 1, 1, 0, 0, 0])
    np.testing.assert_array_equal(want[:, 2], [1, 1, 0, 0, 0, 0])
    np.testing.assert_array_equal(want[:, 3], [1] * 6)


TLE_NET = dict(criterion=dict(name="mse_gain", min_reward=-5))


def test_exploration_settings():
    A = package().algorithms
    assert A.check_exploration(TLE_NET, None) == "imitative"
    assert A.check_exploration(TLE_NET, "imitative") == "imitative"
    assert A.check_exploration(TLE_NET, "greedy") == "greedy"
    # a log-likelihood model ignores the key
    for e in ("greedy", "mixed", "imitation"):
        assert A.check_exploration({}, e) == "imitative"
        assert A.check_exploration(dict(criterion=dict(name="log_likelihood")), e) == "imitative"
    # greedy with weight noise drops dropout (as the reference's noisy graph does), so it runs
    assert A.check_exploration(TLE_NET, "greedy", dict(dropout=True, noise=0.1)) == "greedy"


@pytest.mark.parametrize("exploration, reg, error, message", [
    ("mixed", None, NotImplementedError, "exploration 'mixed'"),
    ("imitation", None, ValueError, "unknown exploration 'imitation'"),
    ("greedy", dict(penalty_coof=0.1), ValueError, "greedy exploration with penalty_coof > 0"),
    ("greedy", dict(dropout=True), NotImplementedError, "greedy exploration with dropout"),
])
def test_exploration_refusals(exploration, reg, error, message):
    """Each refusal is raised by check_exploration and by GradientDescent before any device work."""
    pkg = package()
    with pytest.raises(error, match=message):
        pkg.algorithms.check_exploration(TLE_NET, exploration, reg)
    cfg = O.make_config(**SMALL)
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": 40}, input_num_chars={}, eos_label=cfg["eos_label"], num_phonemes=32, dim_dec=128,
        dims_bidir=[128], subsample=[1], conv_n=8, conv_num_filters=10, post_merge_dims=[128],
        post_merge_activation=pkg.Maxout(2), enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent,
        criterion=dict(name="mse_reward"))
    with pytest.raises(error, match=message):
        pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]),
                            regularization=reg, exploration=exploration)
    # adaptive noise trains the clean graph: the regularisers, and so their refusals, are dropped
    if reg:
        algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]),
                                   regularization=reg, exploration=exploration, adaptive_noise=dict(num_examples=10))
        assert algo.exploration == "greedy"


class _Stop(Exception):
    pass


def _compat_main():
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.main as main
    return main


def _tle_config(tmp_path, training=None, regularization=None):
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as C
    exp = write_experiment(tmp_path)
    cfg = C.Configuration(exp["child"], "$LVSR/lvsr/configs/schema.yaml",
                          [("net.criterion", "{name: mse_gain, min_reward: -5}")])
    cfg = cfg.ordered_stages["main"] if cfg.multi_stage else cfg
    cfg["training"].update(training or {})
    cfg["regularization"] = dict(cfg.get("regularization") or {}, **(regularization or {}))
    return cfg


@pytest.mark.parametrize("exploration", ["greedy", "imitative", None])
def test_compat_train_hands_exploration_through(tmp_path, monkeypatch, exploration):
    main = _compat_main()
    seen = {}

    def fake_descent(**kw):
        seen.update(kw)
        raise _Stop()
    monkeypatch.setattr(main, "create_model", lambda config, data, params: object())
    monkeypatch.setattr(main.pkg, "GradientDescent", fake_descent)
    cfg = _tle_config(tmp_path, training={} if exploration is None else dict(exploration=exploration))
    with pytest.raises(_Stop):
        main.train(cfg, str(tmp_path / "model"))
    assert seen.get("exploration", "imitative") == (exploration or "imitative")


def test_compat_train_refuses_before_the_data(tmp_path, monkeypatch):
    main = _compat_main()

    def no_data(**kw):
        raise AssertionError("the data was built before the refusal")
    monkeypatch.setattr(main, "Data", no_data)
    cfg = _tle_config(tmp_path, training=dict(exploration="greedy"), regularization=dict(penalty_coof=0.5))
    with pytest.raises(ValueError, match="penalty_coof"):
        main.train(cfg, str(tmp_path / "model"))
    cfg = _tle_config(tmp_path, training=dict(exploration="mixed"))
    with pytest.raises(NotImplementedError, match="mixed"):
        main.train(cfg, str(tmp_path / "model"))
