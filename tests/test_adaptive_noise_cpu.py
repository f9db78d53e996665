"""Adaptive weight noise (regularization.adaptive_noise, lvsr/graph.py:71-251) on the host: the float64 oracle's
hand-worked known answer and its ls2 gradient against autograd, the Blocks names of the noise parameters, the
regularization mapping of GradientDescent and a three-stage compat run (GPU calls replaced by recording fakes)."""
import io
import logging
import os
import sys
import tarfile
from collections import OrderedDict

import numpy as np
import pytest

import adaptive_noise_oracle as AN
from compat_helpers import COMPAT, write_experiment
from helpers import package


def test_oracle_known_answer_two_tiny_parameters():
    """x = [1, 3], y = [2], every ls2 = 0 (s2 = 1), coef = 1, N = 1, task gradient [0.1, -0.2 | 0.3], worked by hand:
    prior_u = 6 / 3 = 2; sum (p - u)^2 = 2; prior_s2 = (3 + 2) / 3 = 5 / 3;
    LC = 0.5 * 3 log(5/3) + (2 + 3 - 3 * 5/3) / (2 * 5/3) = 1.5 log(5/3);
    grad p = (p - 2) * 3/5 + g = [-0.5, 0.4 | 0.3];
    grad ls2 = 1024 (3/5 - 1) + 1024 g^2 = [-409.6 + 10.24, -409.6 + 40.96 | -409.6 + 92.16]."""
    params = OrderedDict([("/x.W", np.array([1.0, 3.0])), ("/y.b", np.array([2.0]))])
    ls2 = OrderedDict([("/x.W", np.zeros(2)), ("/y.b", np.zeros(1))])
    lc, u, ps2 = AN.model_cost(params, ls2, num_examples=1, coef=1.0)
    assert u == pytest.approx(2.0, abs=1e-15) and ps2 == pytest.approx(5.0 / 3.0, rel=1e-15)
    assert lc == pytest.approx(1.5 * np.log(5.0 / 3.0), rel=1e-14)
    g = OrderedDict([("/x.W", np.array([0.1, -0.2])), ("/y.b", np.array([0.3]))])
    gp, gl = AN.transform(params, ls2, g, num_examples=1, coef=1.0)
    np.testing.assert_allclose(gp["/x.W"], [-0.5, 0.4], rtol=1e-14)
    np.testing.assert_allclose(gp["/y.b"], [0.3], rtol=1e-14)
    np.testing.assert_allclose(gl["/x.W"], [-399.36, -368.64], rtol=1e-12)
    np.testing.assert_allclose(gl["/y.b"], [-317.44], rtol=1e-12)
    # coef and N scale the model-cost parts only
    gp2, gl2 = AN.transform(params, ls2, g, num_examples=4, coef=0.5)
    np.testing.assert_allclose(gp2["/x.W"], [-1 * 0.6 / 8 + 0.1, 0.6 / 8 - 0.2], rtol=1e-13)
    np.testing.assert_allclose(gl2["/y.b"], [-409.6 / 8 + 92.16], rtol=1e-12)


def test_oracle_gradients_equal_autograd_of_the_model_cost_with_the_priors_held_constant():
    """grad ls2 - 0.5 S s2 g^2 and grad p - g are the derivatives of LC with prior_u, prior_s2 held constant
    (graph.py:238-247), on random parameters of three shapes."""
    import torch
    rng = np.random.RandomState(3)
    params = OrderedDict([("/a.W", rng.normal(size=(3, 4)) * 0.3), ("/b.b", rng.normal(size=5) * 0.1),
                          ("/c.state_to_state", rng.normal(size=(2, 2)))])
    ls2 = OrderedDict((k, np.log(rng.uniform(0.01, 0.2, size=v.shape)) / 1024) for k, v in params.items())
    N, coef = 7, 0.3
    _, u, ps2 = AN.model_cost(params, ls2, N, coef)
    tl = OrderedDict((k, torch.tensor(v, dtype=torch.float64, requires_grad=True)) for k, v in ls2.items())
    tp = OrderedDict((k, torch.tensor(v, dtype=torch.float64, requires_grad=True)) for k, v in params.items())
    lc = 0.0
    for k in params:
        s2 = torch.exp(AN.LOG_SIGMA_SCALE * tl[k])
        lc = lc + 0.5 * (np.log(ps2) - AN.LOG_SIGMA_SCALE * tl[k]).sum() + ((tp[k] - u) ** 2 + s2 - ps2).sum() / (2 * ps2)
    lc = lc / N * coef
    assert float(lc.detach()) == pytest.approx(AN.model_cost(params, ls2, N, coef)[0], rel=1e-12)
    grads = torch.autograd.grad(lc, list(tp.values()) + list(tl.values()))
    zero = OrderedDict((k, np.zeros_like(v)) for k, v in params.items())
    gp, gl = AN.transform(params, ls2, zero, N, coef)
    for (k, _), want in zip(params.items(), grads[:len(params)]):
        np.testing.assert_allclose(gp[k], want.numpy(), rtol=1e-12, atol=1e-15)
    for (k, _), want in zip(params.items(), grads[len(params):]):
        np.testing.assert_allclose(gl[k], want.numpy(), rtol=1e-10, atol=1e-12)


def _blocks_name(brick_path, param_name):
    """graph.py:57-68 (__get_name: the owner's brick path joined by '/', no leading slash, '.', the variable name)
    and B/select.py:199-220 (Selector.get_parameters: '/' + the top brick's path + '.' + the variable name)."""
    noise_var_name = "{}.{}".format("/".join(brick_path), param_name)
    return "/" + "adaptive_noise" + "." + noise_var_name


def test_checkpoint_names_of_the_noise_parameters():
    pkg = package()
    want = "/adaptive_noise.recognizer/encoder/bidir0/forward/fork/fork_inputs.W"
    path = ["recognizer", "encoder", "bidir0", "forward", "fork", "fork_inputs"]
    assert _blocks_name(path, "W") == want
    assert pkg.algorithms.noise_parameter_name("/recognizer/encoder/bidir0/forward/fork/fork_inputs.W") == want
    assert AN.noise_name("/recognizer/encoder/bidir0/forward/fork/fork_inputs.W") == want
    rec = ["recognizer", "generator", "att_trans", "transition"]
    assert pkg.algorithms.noise_parameter_name("/recognizer/generator/att_trans/transition.state_to_gates") == \
        _blocks_name(rec, "state_to_gates")
    # blocks.serialization stores '/' as '|' in the npz keys (serialization.py:606-610)
    assert want.replace("/", "|") == "|adaptive_noise.recognizer|encoder|bidir0|forward|fork|fork_inputs.W"


class _Rec(object):
    lm = None


def test_regularization_mapping_drops_decay_with_the_reference_error(caplog):
    pkg = package()
    with caplog.at_level(logging.ERROR):
        algo = pkg.GradientDescent(recognizer=_Rec(), step_rule=pkg.step_rule_from_config(
            dict(gradient_threshold=10.0, rules=["momentum"], scale=0.1, momentum=0.9)), decay=0.01,
            adaptive_noise=dict(num_examples=3696, model_cost_coefficient=0.1, init_sigma=1e-12))
    assert "weight decay is probably stupid" in caplog.text
    assert algo._tc.decay == 0.0
    assert algo.adaptive_noise == dict(num_examples=3696, init_sigma=1e-12, model_cost_coefficient=0.1, seed=1)
    # the reference's defaults (graph.py:71-80); seed None or 0 is Blocks' default_seed
    algo = pkg.GradientDescent(recognizer=_Rec(), adaptive_noise=dict(num_examples=5, seed=0))
    assert algo.adaptive_noise == dict(num_examples=5, init_sigma=1e-6, model_cost_coefficient=1.0, seed=1)
    assert pkg.GradientDescent(recognizer=_Rec(), decay=0.01)._tc.decay == pytest.approx(0.01)
    with pytest.raises(ValueError):
        pkg.GradientDescent(recognizer=_Rec(), adaptive_noise=dict(init_sigma=1e-6))
    with pytest.raises(TypeError):
        pkg.GradientDescent(recognizer=_Rec(), adaptive_noise=dict(num_examples=5, sigma=1e-6))


STAGES_YAML = """
parent: {base}
training:
    num_batches: 2
stages:
    pretraining:
        number: 0
    main:
        number: 1
        regularization:
            max_norm: 0
            decay: 0.001
            adaptive_noise:
                model_cost_coefficient: 0.1
                init_sigma: 1.0e-12
    annealing:
        number: 2
        regularization:
            max_norm: 0
            adaptive_noise:
                model_cost_coefficient: 0.1
                init_sigma: 1.0e-12
        training:
            scale: 0.1
"""


def test_compat_three_stage_run_saves_and_reloads_the_noise_parameters(tmp_path, monkeypatch, caplog):
    """nips_baseline's stages on the host: `main` trains with adaptive noise from a pretraining checkpoint without
    noise parameters (logged as missing, they keep init_sigma) and saves them into its tar under the Blocks names;
    `annealing` loads them value for value.  The GPU calls are replaced by recording fakes."""
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as LC
    import lvsr.main as M
    pkg = package()
    exp = write_experiment(tmp_path)
    cfg_path = os.path.join(str(tmp_path), "stages.yaml")
    with open(cfg_path, "w") as f:
        f.write(STAGES_YAML.format(base=exp["base"]))
    cfg = LC.Configuration(cfg_path, "$LVSR/lvsr/configs/schema.yaml", [])
    names = ["/recognizer/encoder/bidir0/forward/fork/fork_inputs.W", "/recognizer/generator/readout/post_merge/bias.b"]
    made = []

    class FakeRecognizer(object):
        lm = None

        def __init__(self, load_path):
            self.values = OrderedDict((n, np.full((2, 3) if n.endswith(".W") else (3,), len(made), np.float32))
                                      for n in names)
            self.load_path = load_path

        def get_parameter_values(self):
            return self.values

        save_params = pkg.SpeechRecognizer.save_params
        load_checkpoint_values = staticmethod(pkg.SpeechRecognizer.load_checkpoint_values)

    class FakeGD(object):
        def __init__(self, recognizer, step_rule, decay, adaptive_noise):
            self.recognizer, self.decay, self.adaptive_noise = recognizer, decay, adaptive_noise
            self.noise = OrderedDict((pkg.algorithms.noise_parameter_name(n), np.full(v.shape, -0.027, np.float32))
                                     for n, v in recognizer.values.items())
            self.loaded = None
            made.append(self)

        def initialize(self):
            pass

        def process_batch(self, batch):
            self.last_cost = np.float32(1.5)
            if self.adaptive_noise:
                for v in self.noise.values():
                    v -= 0.001

        def total_gradient_norm(self):
            return 0.5

        def noise_stats(self):
            return dict(model_cost=0.25, model_prior_mean=0.0, model_prior_variance=1e-3)

        def noise_parameter_values(self):
            return OrderedDict((k, v.copy()) for k, v in self.noise.items())

        def set_noise_parameter_values(self, values):
            self.loaded = OrderedDict((k, np.array(v)) for k, v in values.items())
            self.noise.update((k, v.copy()) for k, v in self.loaded.items())

    monkeypatch.setattr(M, "create_model", lambda config, data, load_path=None, test_tag=False: FakeRecognizer(load_path))
    monkeypatch.setattr(M.pkg, "GradientDescent", FakeGD)
    out = os.path.join(str(tmp_path), "run")
    with caplog.at_level(logging.INFO):
        M.train_multistage(cfg, out, "", None, None)
    pre, main, ann = made
    assert pre.adaptive_noise is None and main.recognizer.load_path == os.path.join(out, "pretraining.tar")
    assert main.adaptive_noise == dict(model_cost_coefficient=0.1, init_sigma=1e-12, num_examples=10)
    assert main.decay == pytest.approx(0.001)          # GradientDescent drops it and logs the reference's error
    assert main.loaded == {}                           # pretraining saved no noise parameters
    assert "missing values for parameters" in caplog.text and "model_cost 0.250000" in caplog.text
    with tarfile.open(os.path.join(out, "main.tar")) as tar:
        keys = set(np.load(io.BytesIO(tar.extractfile("_parameters").read())).files)
    assert "|adaptive_noise.recognizer|encoder|bidir0|forward|fork|fork_inputs.W" in keys
    assert "|recognizer|encoder|bidir0|forward|fork|fork_inputs.W" in keys
    with tarfile.open(os.path.join(out, "pretraining.tar")) as tar:
        assert not any("adaptive_noise" in k for k in np.load(io.BytesIO(tar.extractfile("_parameters").read())).files)
    assert list(ann.loaded) == list(main.noise)
    for k, v in main.noise.items():
        assert np.array_equal(ann.loaded[k], v), k
