"""Dropout, weight noise and the alignment penalty on the GPU (regularization.dropout / noise / penalty_coof;
include/lvsr_b200.h): the replayed dropout multiplier and weight-noise eps, the regularised cost and every gradient
against the float64 oracle (tests/regularization_oracle.py) on those draws, the penalty sum against the oracle and the
validation statistic, two optimizer steps, replay and off-settings bit for bit, inference on the means, the padded
frames, and the kernel classes."""
import ctypes as C
from collections import OrderedDict

import numpy as np
import pytest

import bottom_oracle as BO
import content_oracle as CO
import regularization_oracle as RO
from helpers import O, f32, make_recognizer, package
from oracle import lvsr_oracle_grad as G
from test_gpu_bottom import SMALL, _params, _recognizer

pytestmark = pytest.mark.gpu

PYR = dict(SMALL, dims_bidir=[128, 128], subsample=[1, 2])
MEDIAN = dict(type="window_around_median", before=5, after=7)
LEVEL = 0.05
COOF = 0.5


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _rec(cfg, params):
    return _recognizer(cfg, params) if cfg.get("bottom") else make_recognizer(cfg, params)


def _algorithm(rec, reg, tc=None):
    pkg = package()
    rule = pkg.step_rule_from_config(tc, dict(max_norm=tc["max_norm"])) if tc else pkg.CompositeRule([pkg.RemoveNotFinite(0.0)])
    algo = pkg.GradientDescent(recognizer=rec, step_rule=rule, regularization=reg)
    algo.initialize()
    return algo


def _mask(algo, update, offset, T, B, F):
    torch = _torch()
    rec = algo.recognizer
    buf = torch.full((T, B, F), 7.0, dtype=torch.float32, device=rec.device)
    lib = package()._lib.load()
    package()._lib.check(lib.lvsr_train_dropout_mask(rec._require_ready(), update, offset, T, B, F, buf.data_ptr(),
                                                     rec._stream()))
    return buf.cpu().numpy()


def _eps(algo, update):
    """(flat eps of `update`, {parameter name: eps})."""
    torch = _torch()
    rec = algo.recognizer
    buf = torch.full((algo._n,), 7.0, dtype=torch.float32, device=rec.device)
    lib = package()._lib.load()
    package()._lib.check(lib.lvsr_train_weight_noise_sample(rec._require_ready(), update, buf.data_ptr(), rec._stream()))
    flat = buf.cpu().numpy()
    shapes = rec.parameter_shapes()
    return flat, OrderedDict((k, flat[o:o + c].reshape(shapes[k]).astype(np.float64)) for k, (o, c) in algo._offsets().items())


def _draws(algo, cfg, reg, update, batch):
    x = batch[0]
    F = cfg["bottom"]["dims"][-1] if cfg.get("bottom") else cfg["num_features"]
    mult = _mask(algo, update, 0, x.shape[0], x.shape[1], F).astype(np.float64) if reg.get("dropout") else None
    eps = _eps(algo, update)[1] if reg.get("noise") else None
    return mult, eps


def _params_of(cfg, seed):
    if cfg.get("bottom"):
        return _params(cfg, seed)
    init = CO.init_params if cfg.get("attention_type") == "content" else O.init_params
    return OrderedDict((k, f32(v)) for k, v in init(cfg, seed=seed, scale=10.0).items())


def test_dropout_multiplier_is_zero_or_two_fresh_per_update_and_keyed_by_global_utterance():
    _torch()
    cfg = O.make_config(**PYR)
    algo = _algorithm(make_recognizer(cfg, _params_of(cfg, 1)), dict(dropout=True, seed=3))
    T, B, F = 125, 32, 256                                    # 1,024,000 elements
    m0 = _mask(algo, 0, 0, T, B, F)
    assert set(np.unique(m0)) == {0.0, 2.0}
    kept, n = float((m0 > 0).mean()), m0.size
    assert abs(kept - 0.5) < 5 * 0.5 / np.sqrt(n), kept
    m1 = _mask(algo, 1, 0, T, B, F)
    assert abs(np.corrcoef(m0.ravel(), m1.ravel())[0, 1]) < 5 / np.sqrt(n)
    # neighbouring features, frames and utterances are uncorrelated
    assert abs(np.corrcoef(m0[:, :, :-1].ravel(), m0[:, :, 1:].ravel())[0, 1]) < 6 / np.sqrt(n)
    assert abs(np.corrcoef(m0[:-1].ravel(), m0[1:].ravel())[0, 1]) < 6 / np.sqrt(n)
    assert abs(np.corrcoef(m0[:, :-1].ravel(), m0[:, 1:].ravel())[0, 1]) < 6 / np.sqrt(n)
    # a shard at offset 8 draws the columns 8.. of the whole batch, whatever its length
    assert np.array_equal(_mask(algo, 0, 8, T, 4, F), m0[:, 8:12])
    assert np.array_equal(_mask(algo, 0, 8, 60, 4, F), m0[:60, 8:12])
    other = _algorithm(make_recognizer(cfg, _params_of(cfg, 1)), dict(dropout=True, seed=4))
    assert abs(np.corrcoef(m0.ravel(), _mask(other, 0, 0, T, B, F).ravel())[0, 1]) < 5 / np.sqrt(n)


@pytest.mark.parametrize("attention_type", ["content_and_conv", "content"])
def test_weight_noise_eps_is_standard_normal_outside_the_attention_and_zero_inside(attention_type):
    _torch()
    cfg = (CO.make_config(**PYR) if attention_type == "content" else O.make_config(**PYR))
    algo = _algorithm(make_recognizer(cfg, _params_of(cfg, 1)), dict(noise=LEVEL, seed=5))
    flat0, e0 = _eps(algo, 0)
    flat1, _ = _eps(algo, 1)
    inside = np.zeros(algo._n, bool)
    for o, c in algo._offsets().values():
        inside[o:o + c] = True
    assert not flat0[~inside].any()
    subj = np.concatenate([v.ravel() for k, v in e0.items() if RO.is_noise_subject(k)])
    assert all(not v.any() for k, v in e0.items() if not RO.is_noise_subject(k))
    assert any(not RO.is_noise_subject(k) for k in e0)
    n = subj.size
    assert abs(subj.mean()) < 5 / np.sqrt(n) and abs(subj.var() - 1) < 5 * np.sqrt(2.0 / n), (subj.mean(), subj.var())
    for k, v in e0.items():
        if RO.is_noise_subject(k) and v.size >= 4096:
            assert abs(v.mean()) < 5 / np.sqrt(v.size) and abs(v.std() - 1) < 5 / np.sqrt(2 * v.size), k
    f0, f1 = flat0[inside], flat1[inside]
    live = f0 != 0
    assert abs(np.corrcoef(f0[live], f1[live])[0, 1]) < 5 / np.sqrt(live.sum())


def _cases():
    conv = O.make_config(**PYR)
    pen = dict(penalty_coof=COOF)
    return [
        ("penalty_conv", conv, pen, 3),
        ("penalty_logistic", O.make_config(**dict(PYR, energy_normalizer="logistic")), pen, 3),
        ("penalty_relu", O.make_config(**dict(PYR, energy_normalizer="relu")), pen, 2),
        ("penalty_content", CO.make_config(**PYR), pen, 3),
        ("penalty_median_prior", O.make_config(**dict(PYR, prior=MEDIAN)), pen, 3),
        ("noise_conv", conv, dict(noise=LEVEL), 3),
        ("noise_content", CO.make_config(**PYR), dict(noise=LEVEL), 3),
        ("noise_logistic", O.make_config(**dict(PYR, energy_normalizer="logistic")), dict(noise=LEVEL), 2),
        ("dropout_conv", conv, dict(dropout=True), 3),
        ("dropout_bottom_relu", BO.make_config(conv, [256, 100], "relu"), dict(dropout=True), 3),
        ("dropout_bottom_tanh", BO.make_config(CO.make_config(**PYR), [128], "tanh"), dict(dropout=True), 2),
        ("dropout_penalty_median_prior", O.make_config(**dict(PYR, prior=MEDIAN)), dict(dropout=True, **pen), 3),
        ("noise_penalty_logistic", O.make_config(**dict(PYR, energy_normalizer="logistic")), dict(noise=LEVEL, **pen), 2),
        ("dropout_penalty_bottom_batch1", BO.make_config(conv, [128], "tanh"), dict(dropout=True, **pen), 1),
        ("noise_penalty_content_bottom", BO.make_config(CO.make_config(**PYR), [128], "tanh"), dict(noise=LEVEL, **pen), 3),
    ]


def _check(cfg, params, batch, cost, grads, mult, eps, coof=0.0, tol=1e-4, atol_frac=1e-6):
    want_cost, want = RO.cost_and_grads(cfg, params, *batch, mult=mult, eps=eps, level=LEVEL, coof=coof)
    gmax = max(np.abs(w).max() for w in want.values())
    assert list(grads) == list(want)
    bad = {}
    for k, w in want.items():
        e = float(np.abs(grads[k].astype(np.float64) - w).max() / max(np.abs(w).max(), 1e-30))
        if e > tol + atol_frac * gmax / max(np.abs(w).max(), 1e-30):
            bad[k] = e
    assert abs(cost - want_cost) <= 1e-4 * abs(want_cost), (cost, want_cost)
    assert not bad, bad


@pytest.mark.parametrize("name,cfg,reg,B", _cases(), ids=[c[0] for c in _cases()])
def test_regularised_cost_and_gradients_match_the_oracle(name, cfg, reg, B):
    """On a ragged batch: the cost and every parameter's gradient at the replayed draws of update 0 (and the clean
    oracle differs: the regulariser acted)."""
    _torch()
    params = _params_of(cfg, 21)
    batch = O.synthetic_batch(cfg, B=B, T=40, seed=22)
    if cfg.get("bottom"):
        assert not BO.kinks(cfg, params, batch[0], batch[1]), name
    if B > 1:
        assert (batch[1] == 0).any()
    algo = _algorithm(_rec(cfg, params), dict(reg, seed=9))
    cost, grads = algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
    mult, eps = _draws(algo, cfg, reg, 0, batch)
    p64 = OrderedDict((k, v.astype(np.float64)) for k, v in params.items())
    coof = reg.get("penalty_coof", 0.0)
    _check(cfg, p64, batch, cost, grads, mult, eps, coof)
    if coof:
        # the penalty sum of the forward, through the step buffer's slot, against the oracle's
        _, _, want_pen, _ = RO.cost_and_grads(cfg, p64, *batch, mult=mult, eps=eps, level=LEVEL, return_penalty=True)
        got_pen = float(algo._buf[algo._n + 2].item())
        assert want_pen > 0 and abs(got_pen - want_pen) <= 1e-4 * want_pen + 1e-5, (got_pen, want_pen)
    _, clean = RO.cost_and_grads(cfg, p64, *batch)
    assert any(np.abs(clean[k] - grads[k]).max() > 1e-2 * np.abs(clean[k]).max() for k in clean)


def test_two_optimizer_steps_match_the_oracle():
    """process_batch twice with weight noise and the penalty (momentum + AdaDelta + clipping + max-norm): cost,
    last_penalty, gradient norm and every parameter after each step against the oracle's updates of the clean
    parameters."""
    _torch()
    cfg = BO.make_config(O.make_config(**dict(PYR, prior=MEDIAN)), [128], "tanh")
    params = _params_of(cfg, 31)
    tc = G.make_train_config(gradient_threshold=2.0, scale=0.05, momentum=0.5, decay_rate=0.95, epsilon=1e-6,
                             max_norm=1.0)
    reg = dict(noise=LEVEL, penalty_coof=COOF)
    rec = _rec(cfg, params)
    algo = _algorithm(rec, dict(reg, seed=2), tc)
    ref = OrderedDict((k, v.astype(np.float64)) for k, v in params.items())
    state = {}
    for step in range(2):
        batch = O.synthetic_batch(cfg, B=3, T=40, seed=100 + step)
        mult, eps = _draws(algo, cfg, reg, step, batch)
        _, _, pen, _ = RO.cost_and_grads(cfg, ref, *batch, mult=mult, eps=eps, level=LEVEL, return_penalty=True)
        ref, ref_cost, ref_grads = RO.train_step(cfg, ref, state, batch, tc, mult=mult, eps=eps, level=LEVEL, coof=COOF)
        algo.process_batch(dict(zip(algo.SOURCES, batch)))
        assert abs(float(algo.last_cost.item()) - ref_cost) <= 1e-4 * abs(ref_cost), step
        assert abs(float(algo.last_penalty.item()) - pen / 3) <= 1e-4 * pen / 3 + 1e-6, step
        norm = G.l2_norm(ref_grads.values())
        assert abs(algo.total_gradient_norm() - norm) <= 1e-4 * norm, step
        got = rec.get_parameter_values()
        for k, v in ref.items():
            assert np.abs(got[k] - v).max() <= 2e-5 * max(1.0, np.abs(v).max()) + 1e-6, (step, k)


def test_replay_and_off_settings_are_bit_identical_and_inference_reads_the_means():
    torch = _torch()
    pkg = package()
    lib = pkg._lib.load()
    cfg = BO.make_config(O.make_config(**PYR), [128], "relu")
    params = _params_of(cfg, 41)
    batch = dict(zip(pkg.GradientDescent.SOURCES, O.synthetic_batch(cfg, B=3, T=40, seed=42)))
    c_plain, g_plain = _algorithm(_rec(cfg, params), None).cost_and_gradients(batch)
    rec = _rec(cfg, params)
    algo = _algorithm(rec, dict(noise=LEVEL, penalty_coof=COOF, seed=4))
    # all three at once through the C ABI (GradientDescent drops dropout beside noise, as the reference does)
    cfg_all = pkg._lib.LvsrRegularization(dropout=1, noise_level=LEVEL, penalty_coof=COOF, seed=4)
    pkg._lib.check(lib.lvsr_train_set_regularization(rec._require_ready(), C.byref(cfg_all)))
    c1, g1 = algo.cost_and_gradients(batch)
    c2, g2 = algo.cost_and_gradients(batch)               # no update in between: the same draws
    assert c1 == c2 and all(np.array_equal(g1[k], g2[k]) for k in g1)
    assert c1 != c_plain
    # dropout off, level 0 and coefficient 0 set through the C ABI: the step of no regularisation, bit for bit
    off = _algorithm(_rec(cfg, params), None)
    cfg_off = pkg._lib.LvsrRegularization(dropout=0, noise_level=0.0, penalty_coof=0.0, seed=4)
    pkg._lib.check(lib.lvsr_train_set_regularization(off.recognizer._require_ready(), C.byref(cfg_off)))
    c0, g0 = off.cost_and_gradients(batch)
    assert c0 == c_plain and all(np.array_equal(g0[k], g_plain[k]) for k in g0)
    # after a step inference reads the means: cost, validation statistics and beam search equal a fresh model with
    # the same parameters
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=40, seed=43)
    algo.process_batch(batch)
    algo.cost_and_gradients(batch)                        # a training forward between updates changes nothing
    fresh = _rec(cfg, rec.get_parameter_values())
    assert np.array_equal(rec.cost(x, m, labels, lm), fresh.cost(x, m, labels, lm))
    v0, v1 = rec.validation_statistics(x, m, labels, lm), fresh.validation_statistics(x, m, labels, lm)
    assert sorted(v0) == sorted(v1)
    for k in v0:
        assert np.array_equal(np.asarray(v0[k]), np.asarray(v1[k])), k
    utt = {"recordings": x[:int(m[:, 0].sum()), 0]}
    rec.init_beam_search(3)
    fresh.init_beam_search(3)
    a, b = rec.beam_search(dict(utt)), fresh.beam_search(dict(utt))
    assert [list(o) for o in a[0]] == [list(o) for o in b[0]] and np.array_equal(a[1], b[1])
    # the kernel classes run only with their regulariser on
    ms, count = C.c_double(), C.c_int64()

    def launches(algo, cls):
        lib.lvsr_profile_read(cls, C.byref(ms), C.byref(count))
        algo.process_batch(batch)
        pkg._lib.check(lib.lvsr_profile_read(cls, C.byref(ms), C.byref(count)))
        return count.value

    lib.lvsr_profile_enable(1)
    try:
        for cls in (b"dropout", b"weight_noise", b"penalty"):
            assert launches(off, cls) == 0, cls
        assert launches(algo, b"dropout") == 2                # the bottom: forward and backward
        assert launches(algo, b"weight_noise") == 1 and launches(algo, b"penalty") == 1
    finally:
        lib.lvsr_profile_enable(0)
    torch.cuda.synchronize()


@pytest.mark.parametrize("bottom", [False, True], ids=["recordings", "bottom"])
def test_padded_frames_do_not_change_cost_or_gradients(bottom):
    _torch()
    base = O.make_config(**PYR)
    cfg = BO.make_config(base, [128], "tanh") if bottom else base
    params = _params_of(cfg, 51)
    x, m, labels, lm = O.synthetic_batch(cfg, B=4, T=40, seed=52)
    assert (m == 0).any()
    zero = np.where(m[:, :, None] > 0, x, 0.0)
    loud = np.where(m[:, :, None] > 0, x, 1e3 * (1 + np.random.RandomState(0).rand(*x.shape)))
    reg = dict(dropout=True, penalty_coof=COOF, seed=6)
    c0, g0 = _algorithm(_rec(cfg, params), reg).cost_and_gradients(dict(zip(package().GradientDescent.SOURCES, (zero, m, labels, lm))))
    c1, g1 = _algorithm(_rec(cfg, params), reg).cost_and_gradients(dict(zip(package().GradientDescent.SOURCES, (loud, m, labels, lm))))
    assert c0 == c1
    for k in g0:
        assert np.array_equal(g0[k], g1[k]), k


@pytest.mark.parametrize("attention_type", ["content_and_conv", "content"])
def test_penalty_sum_equals_the_validation_statistic(attention_type):
    """Without dropout and noise the training forward's penalty sum is weights_penalty of validation_statistics on the
    same batch (lvsr/expressions.py:14-19), and last_penalty is it over B."""
    _torch()
    cfg = CO.make_config(**PYR) if attention_type == "content" else O.make_config(**PYR)
    params = _params_of(cfg, 61)
    x, m, labels, lm = O.synthetic_batch(cfg, B=4, T=40, seed=62)
    rec = _rec(cfg, params)
    want = rec.validation_statistics(x, m, labels, lm)["weights_penalty"]
    algo = _algorithm(rec, dict(penalty_coof=COOF))
    algo.cost_and_gradients(dict(zip(algo.SOURCES, (x, m, labels, lm))))
    got = float(algo._buf[algo._n + 2].item())
    assert want > 0 and abs(got - want) <= 1e-4 * want, (got, want)
    algo.process_batch(dict(zip(algo.SOURCES, (x, m, labels, lm))))
    assert abs(float(algo.last_penalty.item()) - want / 4) <= 1e-4 * want / 4
