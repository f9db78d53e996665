"""Task-loss-estimation training on the GPU against the float64 oracle of tests/tle_grad_oracle.py: the gradients of
both criteria under imitative and greedy exploration on the TIMIT iclr_reward model and a wsj_jan-shaped model, on
content attention, a deep readout, a forward-only encoder and a bottom MLP, on both decoder plans, at one row and above
the persistent decoder's 64 rows; the greedy prediction step by step; two updates of the step rules; the greedy step
under adaptive and weight noise; and compat's two-stage iclr_reward-like run that trains, validates, checkpoints and
searches.  Per parameter, the worst absolute difference is held to 1e-3 of the oracle's largest entry."""
import os
import sys
from collections import OrderedDict

import numpy as np
import pytest

import bottom_oracle as BO
import content_oracle as CO
import readout_oracle as RO
import regularization_oracle as RG
import tle_grad_oracle as TG
import unidirectional_oracle as U
from compat_helpers import COMPAT, write_experiment
from helpers import O, f32, make_recognizer, package
from oracle import lvsr_oracle_grad as G

pytestmark = pytest.mark.gpu

# exp/timit/configs/iclr_reward.yaml: 3 x BiGRU(256), dim_dec 256, matcher 512, content+conv, the logistic normaliser
ICLR = dict(num_features=123, dims_bidir=[256, 256, 256], subsample=[1, 1, 1], dim_dec=256, dim_matcher=512,
            conv_n=100, conv_num_filters=10, num_phonemes=63, post_merge_dims=[256], maxout_pieces=2,
            energy_normalizer="logistic")
# wsj_jan: one-of-N feedback, the window prior, subsampling
WSJ_JAN = dict(num_features=40, dims_bidir=[256, 256, 256, 256], subsample=[1, 1, 2, 2], dim_dec=256, dim_matcher=512,
               conv_n=100, conv_num_filters=10, num_phonemes=32, post_merge_dims=[256], maxout_pieces=2,
               embed_outputs=False, prior=dict(type="window_around_median", before=5, after=7))
MODELS = dict(iclr=ICLR, wsj_jan=WSJ_JAN)
TOL = 1e-3
NOISE = 1e-4                # float32 error of a readout, relative to the largest readout of its row


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _algo(rec, exploration, **kw):
    pkg = package()
    return pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]),
                               exploration=exploration, **kw)


def _config(net, **kw):
    if net.get("bidir", True) is False:
        return U.make_config(**{k: v for k, v in dict(net, **kw).items() if k != "bidir"})
    if net.get("bottom"):
        return BO.make_config(_config({k: v for k, v in net.items() if k != "bottom"}, **kw), net["bottom"],
                              activation="tanh")
    if net.get("attention_type") == "content":
        return CO.make_config(**dict(net, **kw))
    dims = net["post_merge_dims"]
    if len(dims) > 1:
        return RO.make_config(dims, **{k: v for k, v in dict(net, **kw).items() if k != "post_merge_dims"})
    return O.make_config(**dict(net, **kw))


def _params(cfg, seed):
    if cfg.get("bottom"):
        return BO.init_params(cfg, seed=seed, scale=10.0)
    if cfg.get("bidir", True) is False:
        return U.init_params(cfg, seed=seed, scale=10.0)
    if cfg.get("attention_type") == "content":
        return CO.init_params(cfg, seed=seed, scale=10.0)
    if len(cfg["post_merge_dims"]) > 1:
        return RO.init_params(cfg, seed=seed, scale=10.0)
    return O.init_params(cfg, seed=seed, scale=10.0)


def _compare(grads, want, what):
    bad = {}
    for k, w in want.items():
        err = float(np.abs(grads[k].astype(np.float64) - w).max())
        if err > TOL * max(np.abs(w).max(), 1e-30):
            bad[k] = (err, float(np.abs(w).max()))
    assert not bad, (what, bad)


def _check_step(cfg, params, batch, criterion, exploration, p64=None, **algo_kw):
    """One cost_and_gradients call against the oracle; greedy: the prediction first, step by step, then the oracle's
    gradient on that prediction.  p64: the parameters the step ran on (default: params as float32)."""
    extra = {}
    if cfg.get("bottom"):
        extra["bottom"] = dict(dims=cfg["bottom"]["dims"], activation=package().Tanh())
    if cfg.get("bidir", True) is False:
        extra["bidir"] = False
    rec = make_recognizer(cfg, params, criterion=criterion, **extra)
    algo = _algo(rec, exploration, **algo_kw)
    algo.initialize()
    # the step's own gradient buffer: under adaptive noise cost_and_gradients would add the model cost's terms
    algo._forward_backward(dict(zip(algo.SOURCES, batch)), None)
    cost = float(algo._cost.item())
    grads = _flat_to_params(algo, algo._buf[:algo._n].cpu().numpy())
    x, m, labels, lm = batch
    p64 = p64(algo) if callable(p64) else OrderedDict((k, f32(v)) for k, v in params.items())
    if exploration == "greedy":
        pred, pmask = (t.cpu().numpy() for t in algo.last_prediction)
        assert pred.shape == (labels.shape[0] + TG.EXTRA_STEPS, labels.shape[1])
        ro = TG.greedy_readouts(cfg, p64, x, m, pred)
        TG.check_greedy(ro, pred, NOISE * np.abs(ro).max())
        np.testing.assert_array_equal(pmask, TG.prediction_mask(pred, cfg["eos_label"]))
        want_cost, want = TG.cost_and_grads(cfg, p64, x, m, pred, pmask, criterion, groundtruth=labels)
    else:
        want_cost, want = TG.cost_and_grads(cfg, p64, x, m, labels, lm, criterion)
    assert abs(cost - want_cost) <= 1e-4 * abs(want_cost), (cost, want_cost)
    _compare(grads, want, (criterion, exploration))
    return algo


@pytest.mark.parametrize("model", sorted(MODELS))
@pytest.mark.parametrize("exploration", ["imitative", "greedy"])
@pytest.mark.parametrize("min_reward", [-1.0, -5.0])
@pytest.mark.parametrize("name", ["mse_gain", "mse_reward"])
def test_gradients(model, exploration, min_reward, name):
    cfg = _config(MODELS[model])
    params = _params(cfg, seed=3)
    batch = O.synthetic_batch(cfg, B=3, T=40, seed=23)
    _check_step(cfg, params, batch, dict(name=name, min_reward=min_reward), exploration)


@pytest.mark.parametrize("variant", ["content", "deep_readout", "forward_only", "bottom"])
@pytest.mark.parametrize("exploration", ["imitative", "greedy"])
@pytest.mark.parametrize("name", ["mse_gain", "mse_reward"])
def test_gradients_variants(variant, exploration, name):
    net = dict(ICLR, energy_normalizer="softmax")
    if variant == "content":
        net = dict(net, attention_type="content")
    elif variant == "deep_readout":
        net = dict(net, post_merge_dims=[256, 128], post_merge_activation="tanh", maxout_pieces=1)
    elif variant == "forward_only":
        net = dict(net, bidir=False)
    else:                                   # a Tanh bottom MLP [256] in front of the encoder
        net = dict(net, bottom=[256])
    cfg = _config(net)
    params = _params(cfg, seed=4)
    batch = O.synthetic_batch(cfg, B=3, T=32, seed=29)
    _check_step(cfg, params, batch, dict(name=name, min_reward=-5.0), exploration)


@pytest.mark.parametrize("B", [1, 70])
@pytest.mark.parametrize("stepwise", [False, True])
@pytest.mark.parametrize("exploration", ["imitative", "greedy"])
def test_decoder_plans_and_rows(monkeypatch, B, stepwise, exploration):
    """The persistent decoder and the step-wise kernels (LVSR_NO_DEC_SCAN), at one row and above the persistent
    kernel's 64 rows."""
    if stepwise:
        monkeypatch.setenv("LVSR_NO_DEC_SCAN", "1")
    cfg = _config(ICLR)
    params = _params(cfg, seed=5)
    batch = O.synthetic_batch(cfg, B=B, T=24, seed=31)
    _check_step(cfg, params, batch, dict(name="mse_reward", min_reward=-1.0), exploration)


def test_two_updates_match_the_step_rules():
    """Momentum + AdaDelta + max-norm over two imitative mse_gain steps, as the oracle's step rules apply them."""
    pkg = package()
    cfg = _config(ICLR)
    params = _params(cfg, seed=6)
    crit = dict(name="mse_gain", min_reward=-5.0)
    tc = G.make_train_config(gradient_threshold=100.0, scale=0.01, momentum=0.9, max_norm=1.0)
    rec = make_recognizer(cfg, params, criterion=crit)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(tc, dict(max_norm=1.0)))
    ref = OrderedDict((k, f32(v)) for k, v in params.items())
    state = {}
    for step in range(2):
        batch = O.synthetic_batch(cfg, B=3, T=24, seed=40 + step)
        ref, cost, grads = TG.train_step(cfg, ref, state, batch, tc, crit)
        algo.process_batch(dict(zip(algo.SOURCES, batch)))
        assert abs(float(algo.last_cost.item()) - cost) <= 1e-4 * abs(cost), (step, algo.last_cost.item(), cost)
        got = rec.get_parameter_values()
        for k, v in ref.items():
            assert np.abs(got[k] - v).max() <= 2e-5 * max(1.0, np.abs(v).max()) + 1e-6, (step, k)


def _flat_to_params(algo, flat):
    shapes = algo.recognizer.parameter_shapes()
    return OrderedDict((k, flat[o:o + c].reshape(shapes[k]).astype(np.float64)) for k, (o, c) in algo._offsets().items())


def test_greedy_under_adaptive_noise():
    """The prediction is the oracle's greedy output on the noisy parameters the step ran on, and the gradients at them
    match."""
    torch = _torch()

    def noisy(algo):
        buf = torch.zeros((algo._n,), dtype=torch.float32, device=algo.recognizer.device)
        lib = package()._lib.load()
        package()._lib.check(lib.lvsr_train_noise_params(algo.recognizer._require_ready(), buf.data_ptr(),
                                                         algo.recognizer._stream()))
        return _flat_to_params(algo, buf.cpu().numpy())

    cfg = _config(ICLR)
    params = _params(cfg, seed=7)
    batch = O.synthetic_batch(cfg, B=3, T=24, seed=43)
    _check_step(cfg, params, batch, dict(name="mse_gain", min_reward=-5.0), "greedy", p64=noisy,
                adaptive_noise=dict(num_examples=100, init_sigma=1e-2, seed=3))


def test_greedy_under_weight_noise():
    torch = _torch()
    level = 0.05

    def noisy(algo):
        buf = torch.zeros((algo._n,), dtype=torch.float32, device=algo.recognizer.device)
        lib = package()._lib.load()
        package()._lib.check(lib.lvsr_train_weight_noise_sample(algo.recognizer._require_ready(), 0, buf.data_ptr(),
                                                                algo.recognizer._stream()))
        eps = _flat_to_params(algo, buf.cpu().numpy())
        means = OrderedDict((k, f32(v)) for k, v in algo.recognizer.get_parameter_values().items())
        return OrderedDict((k, f32(v)) for k, v in RG.noisy(means, eps, level).items())

    cfg = _config(ICLR)
    params = _params(cfg, seed=8)
    batch = O.synthetic_batch(cfg, B=3, T=24, seed=47)
    _check_step(cfg, params, batch, dict(name="mse_reward", min_reward=-1.0), "greedy", p64=noisy,
                regularization=dict(noise=level, seed=5))


# exp/timit/configs/iclr_reward.yaml's stages at the toy experiment's widths: mse_gain with greedy exploration and the
# logistic normaliser, min_reward -1, then -5 with adaptive weight noise
ICLR_STAGES = """
parent: {base}
net:
    energy_normalizer: logistic
    criterion:
        name: mse_gain
        min_reward: -1
data:
    validation_batch_size: 2
training:
    exploration: greedy
    num_epochs: 1
monitoring:
    validate_every_epochs: 1
    search_every_epochs: 1
stages:
    main:
        number: 0
        training:
            num_batches: 3
    annealing:
        number: 1
        net:
            criterion:
                name: mse_gain
                min_reward: -5
        regularization:
            adaptive_noise:
                init_sigma: 0.01
        training:
            num_batches: 2
"""


def test_compat_iclr_reward_stages_train_validate_checkpoint_and_search(tmp_path, monkeypatch, capsys):
    _torch()
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as LC
    import lvsr.main as M
    exp = write_experiment(tmp_path)
    path = os.path.join(str(tmp_path), "iclr_reward.yaml")
    with open(path, "w") as f:
        f.write(ICLR_STAGES.format(base=exp["base"]))
    cfg = LC.Configuration(path, None, [])
    steps = []
    real = M.pkg.GradientDescent

    class Spy(real):
        def process_batch(self, batch):
            super().process_batch(batch)
            pred, pmask = self.last_prediction
            steps.append((self.exploration, dict(self.recognizer.criterion), bool(self.adaptive_noise),
                          tuple(pred.shape), batch["labels"].shape, float(self.last_cost.item())))

    made = []
    real_create = M.create_model

    def create_model(config, data, load_path=None, test_tag=False):
        rec = real_create(config, data, load_path, test_tag)
        made.append((load_path, rec))
        return rec

    monkeypatch.setattr(M.pkg, "GradientDescent", Spy)
    monkeypatch.setattr(M, "create_model", create_model)
    out = str(tmp_path / "run")
    M.train_multistage(cfg, out, "", None, None)
    assert [s[:3] for s in steps] == [("greedy", dict(name="mse_gain", min_reward=-1), False)] * 3 + \
        [("greedy", dict(name="mse_gain", min_reward=-5), True)] * 2, steps
    for _, _, _, pshape, lshape, cost in steps:
        assert pshape == (lshape[0] + TG.EXTRA_STEPS, lshape[1]) and np.isfinite(cost)
    (main_path, main), (annealing_path, annealing) = made
    assert main_path is None and annealing_path == os.path.join(out, "main.tar")
    files = set(os.listdir(out))
    assert {"main.tar", "annealing.tar"} <= files, files
    for rec in (main, annealing):
        rows = list(rec.training_log.rows.values())
        assert any("valid_sequence_total_cost" in r and np.isfinite(r["valid_sequence_total_cost"]) for r in rows)
        assert any("valid_per" in r for r in rows)
    # the annealing checkpoint carries the trained noise parameters next to the model's
    saved = package().SpeechRecognizer.load_checkpoint_values(os.path.join(out, "annealing.tar"))
    assert any(k.startswith("/adaptive_noise.") for k in saved)
    # search on the trained checkpoint, through compat's entry point
    stage = cfg.ordered_stages["annealing"]
    M.search(stage, None, os.path.join(out, "annealing.tar"), "valid", None, None, None, False, 1)
    printed = capsys.readouterr().out
    assert printed.strip(), "search printed nothing"
