"""Training with the logistic and relu energy normalisers (lvsr/bricks/attention.py:191-213), as the TIMIT
smooth-focus recipe (exp/timit/configs/nips_smooth.yaml) and the WSJ bhd recipes (exp/wsj/configs/wsj_jan_bhd05.yaml)
do: the gradients of every parameter, the energy bias included, against the float64 gradient oracle at the bar of
test_gpu_train.py (1e-4 of each parameter's largest entry plus a floor of 1e-6 of the model's largest), through
every decoder plan the training forward can take, the optimizer steps, adaptive noise, determinism, the relu row
whose window holds no positive energy, and a compat run of the bhd04 path-addressed initialisation.

Relu energies are kept at least 1e-3 from its kink.  Measured on an H100 80GB HBM3 at a 700 W power limit, over every
gradient comparison of this file: 3.1e-5 of a parameter's largest entry at worst, the energy bias aside (below); the
file runs in about 80 s there."""
import io
import os
import sys
import tarfile

import numpy as np
import pytest

import adaptive_noise_oracle as AN
from compat_helpers import COMPAT, write_experiment
from helpers import O, PYRAMID, check_grads, make_recognizer, package, train_like_the_oracle
from oracle import lvsr_oracle_grad as G

pytestmark = pytest.mark.gpu

ATT = "/recognizer/generator/att_trans/conv_att"
BIAS = ATT + "/energy_comp/linear.b"
PRIORS = dict(default=None,
              moving=dict(type="expanding", initial_begin=0, initial_end=6, min_speed=0.7, max_speed=2.2),
              median=dict(type="window_around_median", before=5, after=7),
              mean=dict(type="window_around_mean", before=6, after=6))
ENERGY_BIAS = dict(logistic=-0.5, relu=1.0)
# exp/timit/configs/nips_smooth.yaml on nips_conv / nips_baseline: 3 x BiGRU(256) without subsampling, 63 phonemes
NIPS_SMOOTH = dict(num_features=123, dims_bidir=[256, 256, 256], subsample=[1, 1, 1], dim_dec=256, dim_matcher=512,
                   conv_n=100, conv_num_filters=10, num_phonemes=63, post_merge_dims=[256], maxout_pieces=2)


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _setup(net, prior, normalizer, B, T, seed):
    cfg = O.make_config(prior=prior, energy_normalizer=normalizer, **net)
    params = O.init_params(cfg, seed=seed, scale=10.0)
    params[BIAS][:] = ENERGY_BIAS[normalizer]
    batch = O.synthetic_batch(cfg, B=B, T=T, seed=seed + 20)
    assert batch[1].sum(axis=0).min() < T                     # ragged lengths
    if normalizer == "relu":
        e = O.recognizer_cost(cfg, params, *batch, return_all=True)["energies"]
        inside = e != 0                                       # energies outside the window are exactly 0
        assert np.abs(e[inside]).min() > 1e-3 and (e[inside] < 0).any() and (e > 0).any(axis=-1).all()
    return cfg, params, batch


def _bias_grad_matches(cfg, params, batch, algo):
    """The energy bias's gradient on its own, at check_grads' bar: 1e-4 of its value plus 1e-6 of the model's largest
    gradient entry.  It is a sum of de over every step and window position whose terms largely cancel, so its float32
    error relative to itself is the largest of the model's: 1.7e-4 in the relu cs4 case (2.1e-7 absolute, within the
    floor), 9.2e-6 or less in every other case."""
    cost, grads = algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
    _, want = G.cost_and_grads(cfg, params, *batch)
    gmax = max(np.abs(w).max() for w in want.values())
    assert want[BIAS][0] != 0
    err = abs(grads[BIAS][0] - want[BIAS][0])
    assert err <= 1e-4 * abs(want[BIAS][0]) + 1e-6 * gmax, (grads[BIAS], want[BIAS], gmax)
    print("energy bias gradient %.6e, oracle %.6e, error %.2e of itself" % (grads[BIAS][0], want[BIAS][0],
                                                                            err / abs(want[BIAS][0])))
    return grads


@pytest.mark.parametrize("prior", list(PRIORS))
@pytest.mark.parametrize("normalizer", ["logistic", "relu"])
def test_gradients_match_the_oracle(normalizer, prior):
    """Every parameter at the PYRAMID shape, B = 4 with ragged lengths, each prior; the energy bias on its own."""
    _torch()
    cfg, params, batch = _setup(PYRAMID, PRIORS[prior], normalizer, B=4, T=64, seed=5)
    algo, rec = check_grads(cfg, params, batch)
    _bias_grad_matches(cfg, params, batch, algo)


@pytest.mark.parametrize("plan", ["cs1", "cs2", "cs4", "cs8", "stepwise"])
@pytest.mark.parametrize("normalizer", ["logistic", "relu"])
def test_gradients_through_every_decoder_plan(normalizer, plan, monkeypatch):
    """The training forward forced onto the persistent decoder at each cluster size (LVSR_DEC_CS) and onto the step-wise
    kernels (LVSR_NO_DEC_SCAN): the backward reads the energies each of them wrote.  One BiGRU(128) layer, so T' = T
    and T' reaches the 16 positions per CTA a cluster of 8 needs."""
    _torch()
    for k in ("LVSR_DEC_CS", "LVSR_DEC_LAYOUT", "LVSR_DEC_HANDLER", "LVSR_ATT_CS", "LVSR_NO_DEC_SCAN"):
        monkeypatch.delenv(k, raising=False)
    cs = None if plan == "stepwise" else int(plan[2:])
    if cs is None:
        monkeypatch.setenv("LVSR_NO_DEC_SCAN", "1")
    else:
        monkeypatch.setenv("LVSR_DEC_CS", str(cs))
        monkeypatch.setenv("LVSR_DEC_CHECK", "1")
    Tp = max(16 * (cs or 1), 24) + 3
    net = dict(PYRAMID, dims_bidir=[128], subsample=[1])
    cfg, params, batch = _setup(net, PRIORS["median"], normalizer, B=4, T=Tp, seed=7)
    algo, rec = check_grads(cfg, params, batch)
    got = rec.decoder_plan()
    if cs is None:
        assert not got["ran"] and got["kernel"] == "stepwise", got
    else:
        assert got["ran"] and got["kernel"] == "dec_scan" and got["cs"] == cs, got
    _bias_grad_matches(cfg, params, batch, algo)


def test_nips_smooth_gradients_and_two_optimizer_steps():
    """The smooth-focus TIMIT architecture at T' = 300 frames: gradients, then two updates of its main stage's rules
    (momentum + AdaDelta + max-norm, lvsr/main.py:480-519) equal to the oracle's.  The energy bias has no WEIGHT role:
    max-norm leaves it alone."""
    _torch()
    cfg, params, batch = _setup(NIPS_SMOOTH, None, "logistic", B=4, T=300, seed=3)
    algo, _ = check_grads(cfg, params, batch)
    _bias_grad_matches(cfg, params, batch, algo)
    assert not G.is_weight(BIAS)
    tc = G.make_train_config(gradient_threshold=100.0, rules=("momentum", "adadelta"), scale=0.1, momentum=0.9,
                             decay_rate=0.95, epsilon=1e-8, max_norm=1.0)
    rec, ref, norms = train_like_the_oracle(cfg, params, tc, steps=2, B=4, T=300)
    assert rec.get_parameter_values()[BIAS][0] != ENERGY_BIAS["logistic"]


def test_adaptive_noise_step_with_logistic():
    """One adaptive-noise update (lvsr/graph.py:71-251) with the logistic normaliser against
    tests/adaptive_noise_oracle.py on the replayed noise: the energy bias gets a mean and a log-variance like every
    other parameter."""
    torch = _torch()
    pkg = package()
    cfg, params, batch = _setup(PYRAMID, None, "logistic", B=3, T=32, seed=5)
    tc = G.make_train_config(gradient_threshold=2.0, rules=("momentum", "adadelta"), scale=0.05, momentum=0.5,
                             decay_rate=0.95, epsilon=1e-6, max_norm=1.0)
    rec = make_recognizer(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(tc, dict(max_norm=1.0)),
                               adaptive_noise=dict(num_examples=1000, init_sigma=1e-2, model_cost_coefficient=0.5,
                                                   seed=7))
    algo.initialize()
    lib, h = pkg._lib.load(), rec._require_ready()
    buf = torch.zeros((algo._n,), dtype=torch.float32, device=rec.device)
    pkg._lib.check(lib.lvsr_train_noise_sample(h, 0, buf.data_ptr(), rec._stream()))
    flat = buf.cpu().numpy()
    shapes = rec.parameter_shapes()
    eps = {k: flat[o:o + c].reshape(shapes[k]).astype(np.float64) for k, (o, c) in algo._offsets().items()}
    ref = {k: np.asarray(v, np.float32).astype(np.float64) for k, v in params.items()}
    ls2 = AN.init_ls2(ref, 1e-2)
    ref, ls2, cost, _, norm = AN.train_step(cfg, ref, ls2, {}, batch, tc, eps, 1000, 0.5)
    algo.process_batch(dict(zip(algo.SOURCES, batch)))
    assert abs(float(algo.last_cost.item()) - cost) <= 1e-4 * abs(cost)
    assert abs(algo.total_gradient_norm() - norm) <= 1e-4 * norm
    got, got_ls2 = rec.get_parameter_values(), algo.noise_parameter_values()
    for k, v in ref.items():
        assert np.abs(got[k] - v).max() <= 1e-4 * np.abs(v).max(), k
        assert np.abs(got_ls2[AN.noise_name(k)] - ls2[k]).max() <= 1e-4 * np.abs(ls2[k]).max(), k


@pytest.mark.parametrize("normalizer", ["logistic", "relu"])
def test_two_calls_give_bit_identical_gradients(normalizer):
    _torch()
    pkg = package()
    cfg, params, batch = _setup(PYRAMID, PRIORS["median"], normalizer, B=4, T=64, seed=5)
    algo = pkg.GradientDescent(recognizer=make_recognizer(cfg, params),
                               step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
    c1, g1 = algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
    c2, g2 = algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
    assert c1 == c2 and all(np.array_equal(g1[k], g2[k]) for k in g1)


def test_relu_window_without_a_positive_energy_takes_the_reference_step():
    """Every energy below 0: each relu row's weights are 0 / 0, NaN in the reference (lvsr/bricks/attention.py:211-213)
    and on the GPU.  The gradient is not finite, the clipping multiplier NaN, and RemoveNotFinite(0.0) replaces each
    step by the parameter itself (B/algorithms/__init__.py:855-861): every parameter becomes 0, as the oracle's
    train_step has it.  (The reference's comment there says parameters are left unchanged; its arithmetic zeroes
    them, and lvsr's main loop then stops on the NaN gradient norm, lvsr/main.py:624-626.)"""
    _torch()
    pkg = package()
    cfg = O.make_config(energy_normalizer="relu", **PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    params[BIAS][:] = -100.0
    batch = O.synthetic_batch(cfg, B=3, T=32, seed=25)
    with np.errstate(invalid="ignore"):
        out = O.recognizer_cost(cfg, params, *batch, return_all=True)
    assert (out["energies"][0] < 0).all() and np.isnan(out["costs"]).all()     # NaN from the first step on
    rec = make_recognizer(cfg, params)
    assert not np.isfinite(rec.cost(*batch)).all()
    tc = G.make_train_config(gradient_threshold=1.0, rules=("momentum", "adadelta"), scale=0.1, momentum=0.5,
                             decay_rate=0.95, epsilon=1e-6, max_norm=1.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        ref, _, _ = G.train_step(cfg, params, {}, batch, tc)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(tc, dict(max_norm=1.0)))
    algo.process_batch(dict(zip(algo.SOURCES, batch)))
    assert not np.isfinite(float(algo.last_cost.item()))
    got = rec.get_parameter_values()
    for k, v in ref.items():
        assert np.array_equal(got[k], np.asarray(v, np.float32)), k
    assert not any(v.any() for v in got.values())


BHD_YAML = """
parent: {base}
net:
    dims_bidir: [128, 128, 128]
    subsample: [1, 1, 1]
    energy_normalizer: logistic
initialization:
    /recognizer:
        weights_init:
          !!python/object:blocks.initialization.Uniform {{width: 0.1}}
    /recognizer/generator/att_trans/conv_att/energy_comp:
        weights_init:
          !!python/object/apply:blocks.initialization.Constant [0.]
training:
    num_batches: 2
stages:
    pretraining:
        number: 0
    main:
        number: 1
        training:
            scale: 0.5
"""


def test_compat_bhd04_initialization_trains_and_saves_the_energy_bias(tmp_path, monkeypatch):
    """lvsr.main.train_multistage on a tiny smooth-focus experiment with the initialisation of
    exp/wsj/configs/wsj_jan_bhd04.yaml: energy_comp's weights start at 0, every other weight in U(-0.05, 0.05), and the
    checkpoint holds the trained energy bias."""
    _torch()
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as LC
    import lvsr.main as M
    pkg = package()
    exp = write_experiment(tmp_path)
    path = os.path.join(str(tmp_path), "bhd.yaml")
    with open(path, "w") as f:
        f.write(BHD_YAML.format(base=exp["base"]))
    cfg = LC.Configuration(path, "$LVSR/lvsr/configs/schema.yaml", [])
    drawn = []
    orig = pkg.SpeechRecognizer.initial_values

    def record(self, shapes, seed=1):
        drawn.append(orig(self, shapes, seed))
        return drawn[-1]
    monkeypatch.setattr(pkg.SpeechRecognizer, "initial_values", record)
    out = os.path.join(str(tmp_path), "run")
    M.train_multistage(cfg, out, "", None, None)
    init = drawn[0]
    assert not init[ATT + "/energy_comp/linear.W"].any() and not init[BIAS].any()
    for k, v in init.items():
        leaf = k.rsplit(".", 1)[1]
        if leaf in ("W", "filters") and "energy_comp" not in k:
            assert np.abs(v).max() <= 0.05 and np.abs(v).max() > 0.04, k
    with tarfile.open(os.path.join(out, "main.tar")) as tar:
        data = np.load(io.BytesIO(tar.extractfile("_parameters").read()))
        saved = {k.replace("|", "/"): data[k] for k in data.files}
    assert saved[BIAS].shape == (1,) and saved[BIAS][0] != 0
    assert saved[ATT + "/energy_comp/linear.W"].any()
