"""The bottom MLP (net.bottom.dims) without a GPU: the float64 bottom oracle, its torch mirror and finite differences,
the parameter table and initialisation order, and the configuration plumbing."""
import sys

import numpy as np
import pytest
from numpy.testing import assert_allclose

from oracle import lvsr_oracle as O
import bottom_oracle as BO
import content_oracle as CO
from compat_helpers import COMPAT, write_experiment
from helpers import package

TINY = dict(num_features=6, dims_bidir=[16, 16], subsample=[1, 2], dim_dec=16, dim_matcher=24, conv_n=3,
            conv_num_filters=4, num_phonemes=10, post_merge_dims=[16], maxout_pieces=2)


def test_blocks_mlp_known_answer():
    """libs/blocks/tests/bricks/test_bricks.py:344-354 (test_mlp): MLP([Tanh(), None], [16, 8, 4]) with every weight and
    bias Constant(1) is tanh(x 1 + 1) 1 + 1.  The bottom's layers are that MLP's, with the activation after each one,
    so its first layer is the known answer's hidden layer and the second one's pre-activation its output."""
    rng = np.random.RandomState(0)
    x = rng.rand(2, 16)
    cfg = BO.make_config(O.make_config(num_features=16), [8, 4], "tanh")
    params = {BO.linear_name(0) + ".W": np.ones((16, 8)), BO.linear_name(0) + ".b": np.ones(8),
              BO.linear_name(1) + ".W": np.ones((8, 4)), BO.linear_name(1) + ".b": np.ones(4)}
    want = np.tanh(x.dot(np.ones((16, 8))) + np.ones((2, 8))).dot(np.ones((8, 4))) + np.ones((2, 4))
    assert_allclose(BO.pre_activations(cfg, params, x)[1], want, rtol=1e-12)
    assert_allclose(BO.bottom(cfg, params, x), np.tanh(want), rtol=1e-12)


def test_rectifier_value_and_derivative_at_zero():
    """Rectifier = switch(x > 0, x, 0): 0 at and below 0, and a derivative of 0 at 0 (Theano's gradient of the switch),
    in the numpy oracle and the torch mirror alike."""
    import torch
    assert_allclose(BO.rectifier(np.array([-2.0, -0.0, 0.0, 1e-300, 3.0])), [0, 0, 0, 1e-300, 3.0])
    cfg = BO.make_config(O.make_config(num_features=3), [3], "relu")
    p = {BO.linear_name(0) + ".W": torch.eye(3, dtype=torch.float64, requires_grad=True),
         BO.linear_name(0) + ".b": torch.zeros(3, dtype=torch.float64, requires_grad=True)}
    x = torch.tensor([[0.0, -1.0, 2.0]], dtype=torch.float64, requires_grad=True)
    y = BO._bottom_torch(cfg, p, x)
    (g,) = torch.autograd.grad(y.sum(), [x])
    assert y.tolist() == [[0.0, 0.0, 2.0]]
    assert g.tolist() == [[0.0, 0.0, 1.0]]


def _case(attention_type, dims, activation, seed=3):
    base = CO.make_config(**TINY) if attention_type == "content" else O.make_config(**TINY)
    cfg = BO.make_config(base, dims, activation)
    params = BO.init_params(cfg, seed=seed, scale=10.0)
    rng = np.random.RandomState(seed)
    for i in range(len(dims)):              # non-zero biases: their gradients are checked too
        params[BO.linear_name(i) + ".b"] = rng.normal(0, 0.3, size=dims[i])
    batch = O.synthetic_batch(cfg, B=3, T=12, seed=5)
    return cfg, params, batch


@pytest.mark.parametrize("attention_type,dims,activation", [
    ("content_and_conv", [10], "relu"), ("content_and_conv", [9, 7], "tanh"), ("content", [10, 5], "relu")])
def test_torch_mirror_equals_the_numpy_oracle(attention_type, dims, activation):
    cfg, params, batch = _case(attention_type, dims, activation)
    want = BO.recognizer_cost(cfg, params, *batch)
    _, _, got = BO.cost_and_grads(cfg, params, *batch, return_costs=True)
    assert_allclose(got, want, rtol=0, atol=1e-12)


@pytest.mark.parametrize("attention_type,dims,activation", [
    ("content_and_conv", [10], "relu"), ("content_and_conv", [9, 7], "tanh"), ("content", [10, 5], "relu")])
def test_autograd_matches_finite_differences(attention_type, dims, activation):
    """Central differences of the numpy oracle's cost against the mirror's gradients, at a few entries of every bottom
    parameter and of encoder layer 0's fork (which now reads the bottom's output)."""
    cfg, params, batch = _case(attention_type, dims, activation)
    assert not BO.kinks(cfg, params, batch[0], batch[1], eps=1e-4)
    _, grads = BO.cost_and_grads(cfg, params, *batch)
    rng = np.random.RandomState(0)
    names = [k for k in params if k.startswith(BO.BOTTOM)] + ["/recognizer/encoder/bidir0/forward/fork/fork_inputs.W"]
    h = 1e-6
    for name in names:
        for _ in range(3):
            idx = tuple(rng.randint(s) for s in params[name].shape)
            plus, minus = dict(params), dict(params)
            plus[name] = params[name].copy()
            minus[name] = params[name].copy()
            plus[name][idx] += h
            minus[name][idx] -= h
            fd = (O.batch_cost(BO.recognizer_cost(cfg, plus, *batch)) -
                  O.batch_cost(BO.recognizer_cost(cfg, minus, *batch))) / (2 * h)
            assert abs(fd - grads[name][idx]) <= 1e-6 * max(1.0, abs(fd)), (name, idx, fd, grads[name][idx])
    assert any(np.abs(grads[k]).max() > 0 for k in names if k.startswith(BO.BOTTOM))


# wsj_jan_new.yaml (one-of-N feedback, 4 BiGRU layers of 250, subsampling [1, 1, 2, 2] ...) with bottom.dims [256] at
# the widths the kernels take: BiGRU 256, dim_dec 256, dim_matcher 512, 123 features
WSJ_JAN_NEW = dict(num_features=123, dims_bidir=[256, 256, 256, 256], subsample=[1, 1, 2, 2], dim_dec=256,
                   dim_matcher=512, conv_n=100, conv_num_filters=10, num_phonemes=32, post_merge_dims=[256],
                   maxout_pieces=2, embed_outputs=False)


def test_wsj_jan_new_parameter_table():
    """The bottom's Linear sits after the encoder's 56 parameters and before the generator's, W before b, named
    /recognizer/bottom/bottom/linear_0 (SpeechBottom "bottom" > MLP "bottom" > Linear "linear_0"); encoder layer 0
    takes the bottom's 256 features."""
    cfg = BO.make_config(O.make_config(**WSJ_JAN_NEW), [256], "relu")
    items = list(BO.param_shapes(cfg).items())
    single = list(O.param_shapes(BO.inner(cfg)).items())
    assert items[:56] == single[:56] and all(k.startswith("/recognizer/encoder/") for k, _ in items[:56])
    assert items[56:58] == [("/recognizer/bottom/bottom/linear_0.W", (123, 256)),
                            ("/recognizer/bottom/bottom/linear_0.b", (256,))]
    assert items[58:] == single[56:] and items[58][0].startswith("/recognizer/generator/")
    assert dict(items)["/recognizer/encoder/bidir0/forward/fork/fork_inputs.W"] == (256, 256)


def _recognizer(pkg, **kw):
    return pkg.SpeechRecognizer(input_dims={"recordings": 6}, input_num_chars={}, eos_label=9, num_phonemes=10,
                                dim_dec=16, dims_bidir=[16, 16], subsample=[1, 2], conv_n=3, conv_num_filters=4,
                                dim_matcher=24, post_merge_dims=[16], post_merge_activation=pkg.Maxout(2), **kw)


def test_initialization_walks_the_bottom_in_brick_order():
    """initialize() draws what the oracle's init_params draws on the table with the bottom (weights_init on W,
    biases_init on b, one RandomState in brick order), and a /recognizer/bottom path overrides both for the bottom
    alone; its W carries the WEIGHT role (decay and max-norm)."""
    from oracle import lvsr_oracle_grad as G
    pkg = package()
    cfg = BO.make_config(O.make_config(**TINY), [10, 7], "relu")
    rec = _recognizer(pkg, bottom=dict(dims=[10, 7], activation=pkg.Rectifier()))
    rec.set_initialization("/recognizer", weights_init=pkg.IsotropicGaussian(0.01), biases_init=pkg.Constant(0.0),
                           rec_weights_init=pkg.Orthogonal(), initial_states_init=pkg.IsotropicGaussian(0.001))
    shapes = BO.param_shapes(cfg)
    got = rec.initial_values(shapes, seed=1)
    want = BO.init_params(cfg, seed=1)
    assert list(got) == list(want)
    for k, v in want.items():
        assert_allclose(got[k], v.astype(np.float32), rtol=1e-6, atol=1e-9, err_msg=k)
    rec.set_initialization("/recognizer/bottom", weights_init=pkg.Constant(0.5), biases_init=pkg.Constant(0.25))
    got = rec.initial_values(shapes, seed=1)
    for k in shapes:
        if k.startswith("/recognizer/bottom/"):
            assert np.all(got[k] == (0.5 if k.endswith(".W") else 0.25)), k
        elif k.startswith("/recognizer/encoder/"):      # drawn before the bottom; Constant draws nothing after it
            assert_allclose(got[k], want[k].astype(np.float32), rtol=1e-6, atol=1e-9, err_msg=k)
    assert G.is_weight(BO.linear_name(0) + ".W") and not G.is_weight(BO.linear_name(0) + ".b")


def test_config_plumbing():
    """bottom absent, None and dims [] give today's net and no bottom config; activation None is Tanh; Rectifier and
    Tanh reach lvsr_bottom_config; Maxout and deeper stacks than the struct holds are refused."""
    pkg = package()
    plain = _recognizer(pkg)
    assert plain._make_bottom_config() is None
    for bottom in (None, {}, dict(dims=[], activation=pkg.Rectifier()), dict(dims=None, bottom_class=object)):
        rec = _recognizer(pkg, bottom=bottom)
        assert rec.net == plain.net and rec._make_bottom_config() is None
        assert bytes(rec._make_config()) == bytes(plain._make_config())
    rec = _recognizer(pkg, bottom=dict(dims=[100], activation=None))
    assert rec.net["bottom"] == dict(dims=[100], activation="tanh")
    b = rec._make_bottom_config()
    assert (b.num_layers, b.dims[0], b.activation) == (1, 100, 2)
    rec = _recognizer(pkg, bottom=dict(dims=[250, 64], activation=pkg.Rectifier(), bottom_class=object))
    b = rec._make_bottom_config()
    assert (b.num_layers, list(b.dims)[:2], b.activation) == (2, [250, 64], 1)
    assert bytes(rec._make_config()) == bytes(plain._make_config())      # lvsr_config itself is unchanged
    with pytest.raises(NotImplementedError, match="bottom MLP activation"):
        _recognizer(pkg, bottom=dict(dims=[100], activation=pkg.Maxout(2)))
    with pytest.raises(NotImplementedError, match="bottom MLP of 5 layers"):
        _recognizer(pkg, bottom=dict(dims=[8] * 5, activation=pkg.Tanh()))._make_bottom_config()
    fields = [f for f, _ in pkg._lib.LvsrBottomConfig._fields_]
    assert fields == ["num_layers", "dims", "activation"]


def test_compat_create_model_passes_the_bottom(tmp_path, monkeypatch):
    """compat's create_model hands config['net']['bottom'] from the YAML (bottom_class dropped) to the recognizer."""
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as LC
    import lvsr.main as LM
    from lvsr.datasets import Data
    pkg = package()
    monkeypatch.setattr(pkg.SpeechRecognizer, "initialize", lambda self, seed=1: None)
    exp = write_experiment(tmp_path)
    cfg = LC.Configuration(exp["base"], "$LVSR/lvsr/configs/schema.yaml", [("net.bottom.dims", "[64]")])
    rec = LM.create_model(cfg, Data(**cfg["data"]))
    assert rec.net["bottom"] == dict(dims=[64], activation="relu")
    assert rec.net["num_features"] == 40
