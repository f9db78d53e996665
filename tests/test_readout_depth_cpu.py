"""The deep readout (net.post_merge_dims of 2 to 4 entries) without a GPU: its oracle against the reference's
formulas, the torch mirror against the oracle and against central differences, the host's parameter table and
initialisation, and every refusal of a readout the library does not run, with its message, before any device work."""
import ctypes
import os
import re

import numpy as np
import pytest
from numpy.testing import assert_allclose

from oracle import lvsr_oracle as O
import readout_oracle as RO
from helpers import ROOT, package


def small_cfg(dims, act="tanh", use_states=True, **kw):
    return RO.make_config(dims, num_features=6, dims_bidir=[8], dim_dec=8, dim_matcher=8, conv_n=2, conv_num_filters=2,
                          num_phonemes=5, post_merge_activation=act, maxout_pieces=1,
                          use_states_for_readout=use_states, **kw)


def test_depth_one_is_the_single_layer_readout():
    for act, pieces in (("maxout", 2), ("relu", 1), ("tanh", 1), ("identity", 1)):
        cfg = RO.make_config([16], num_features=6, dims_bidir=[8], dim_dec=8, dim_matcher=8, conv_n=2,
                             conv_num_filters=2, num_phonemes=5, post_merge_activation=act, maxout_pieces=pieces)
        assert RO.param_shapes(cfg) == O.param_shapes(cfg)
        params = RO.init_params(cfg, seed=3, scale=10.0)
        rng = np.random.RandomState(0)
        s, wa = rng.randn(3, 4, 8), rng.randn(3, 4, 16)
        assert_allclose(RO.readout(cfg, params, s, wa), O.readout(cfg, params, s, wa), rtol=0, atol=1e-12)


def blocks_mlp(activations, dims, x, Ws, bs):
    """Blocks' MLP (libs/blocks/blocks/bricks/sequences.py: MLP = Sequence of Linear(dims[i], dims[i+1]) and
    activations[i]) applied as the reference's post_merge applies it, after Bias and the activation."""
    for act, W, b, din, dout in zip(activations, Ws, bs, dims[:-1], dims[1:]):
        assert W.shape == (din, dout) and b.shape == (dout,)
        x = act(x.dot(W) + b)
    return x


@pytest.mark.parametrize("dims,act", [([16, 24], "tanh"), ([16, 8, 32], "relu"), ([8, 8, 16, 24], "identity"),
                                      ([16, 16], "maxout")])
def test_body_is_blocks_mlp(dims, act):
    cfg = small_cfg(dims, act)
    params = RO.init_params(cfg, seed=5, scale=30.0)
    rng = np.random.RandomState(1)
    s, wa = rng.randn(3, 2, 8), rng.randn(3, 2, 16)
    f = {"tanh": np.tanh, "relu": lambda x: np.maximum(x, 0), "identity": lambda x: x, "maxout": lambda x: x}[act]
    merged = wa.dot(params[O._GEN + "/readout/merge/transform_weighted_averages.W"]) + \
        s.dot(params[O._GEN + "/readout/merge/transform_states.W"]) + params[RO.PM + "/bias.b"]
    k = len(dims)
    Ws = [params[RO.linear_name(j) + ".W"] for j in range(k)]
    bs = [params[RO.linear_name(j) + ".b"] for j in range(k)]
    want = blocks_mlp([f] * (k - 1) + [lambda x: x], dims + [cfg["num_phonemes"]], f(merged), Ws, bs)
    assert_allclose(RO.readout(cfg, params, s, wa), want, rtol=0, atol=1e-12)


def test_known_answers():
    # 2-layer Tanh: merged = ctx . Wc (no states), h0 = tanh(merged + b), h1 = tanh(h0 W0 + b0), logits = h1 W1 + b1
    cfg = RO.make_config([8, 8], num_features=6, dims_bidir=[8], dim_dec=8, dim_matcher=8, conv_n=2,
                         conv_num_filters=2, num_phonemes=2, post_merge_activation="tanh", maxout_pieces=1,
                         use_states_for_readout=False)
    p = {k: np.zeros(v) for k, v in RO.param_shapes(cfg).items()}
    p[O._GEN + "/readout/merge/transform_weighted_averages.W"][0, 0] = 1.0       # merged[0] = ctx[0]
    p[RO.PM + "/bias.b"][0] = 0.5
    p[RO.linear_name(0) + ".W"][0, 1] = 2.0                                        # z1[1] = 2 h0[0]
    p[RO.linear_name(0) + ".b"][1] = -1.0
    p[RO.linear_name(1) + ".W"][1, 0] = 3.0                                        # logit 0 = 3 h1[1]
    p[RO.linear_name(1) + ".b"][:] = [0.25, -0.75]
    ctx = np.zeros((1, 16))
    ctx[0, 0] = 0.3
    h0 = np.tanh(0.3 + 0.5)
    h1 = np.tanh(2.0 * h0 - 1.0)
    assert_allclose(RO.readout(cfg, p, None, ctx), [[3.0 * h1 + 0.25, -0.75]], rtol=0, atol=1e-15)
    # 3-layer Rectifier: a negative unit is cut at every layer
    cfg = small_cfg([8, 8, 8], "relu", use_states=False)
    p = {k: np.zeros(v) for k, v in RO.param_shapes(cfg).items()}
    Wc = p[O._GEN + "/readout/merge/transform_weighted_averages.W"]
    Wc[0, 0], Wc[1, 1] = 1.0, -1.0                                                # h0 = relu([c0, -c1, ..])
    p[RO.linear_name(0) + ".W"][0, 0] = 2.0
    p[RO.linear_name(0) + ".W"][1, 1] = 5.0
    p[RO.linear_name(0) + ".b"][1] = -0.5                                          # h1 = relu([2 h0[0], 5 h0[1] - .5])
    p[RO.linear_name(1) + ".W"][0, 0] = 1.0
    p[RO.linear_name(1) + ".W"][1, 0] = 1.0
    p[RO.linear_name(1) + ".b"][0] = -4.0                                          # h2[0] = relu(h1[0] + h1[1] - 4)
    p[RO.linear_name(2) + ".W"][0, 4] = 1.0
    ctx = np.zeros((2, 16))
    ctx[0, :2] = [3.0, -1.0]        # h0 = [3, 1], h1 = [6, 4.5], h2[0] = 6.5
    ctx[1, :2] = [1.0, 2.0]         # h0 = [1, 0], h1 = [2, 0],   h2[0] = 0
    assert_allclose(RO.readout(cfg, p, None, ctx)[:, 4], [6.5, 0.0], rtol=0, atol=1e-15)


@pytest.mark.parametrize("dims,act", [([16, 24], "tanh"), ([16, 8, 16], "relu")])
def test_torch_mirror_and_its_gradient(dims, act):
    torch = pytest.importorskip("torch")
    cfg = small_cfg(dims, act)
    params = RO.init_params(cfg, seed=2, scale=20.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=2, T=10, seed=4)
    cost, grads, costs = RO.cost_and_grads(cfg, params, x, m, labels, lm, return_costs=True)
    want = RO.recognizer_cost(cfg, params, x, m, labels, lm)
    assert_allclose(costs, want, rtol=1e-11, atol=1e-11)
    assert abs(cost - want.sum() / labels.shape[1]) < 1e-11
    rng = np.random.RandomState(0)
    eps = 1e-6
    for name in [RO.PM + "/bias.b"] + [RO.linear_name(j) + leaf for j in range(len(dims)) for leaf in (".W", ".b")]:
        for _ in range(3):
            idx = tuple(rng.randint(n) for n in params[name].shape)
            plus, minus = dict(params), dict(params)
            plus[name] = params[name].copy()
            minus[name] = params[name].copy()
            plus[name][idx] += eps
            minus[name][idx] -= eps
            fd = (RO.recognizer_cost(cfg, plus, x, m, labels, lm).sum() -
                  RO.recognizer_cost(cfg, minus, x, m, labels, lm).sum()) / (2 * eps * labels.shape[1])
            assert abs(fd - grads[name][idx]) <= 1e-6 * max(1.0, abs(fd)), (name, idx, fd, grads[name][idx])


def _kw(pkg, dims, act=None):
    return dict(input_dims={"recordings": 6}, input_num_chars={}, eos_label=4, num_phonemes=5, dim_dec=16,
                dims_bidir=[64], conv_n=3, conv_num_filters=2, post_merge_dims=dims,
                post_merge_activation=act if act is not None else pkg.Rectifier())


def test_parameter_table_and_initialisation():
    """The host's draws over the deep table are O.init_params's scheme walked in brick order; a scheme pushed onto
    /post_merge/mlp reaches every Linear of the MLP and nothing else."""
    pkg = package()
    cfg = RO.make_config([16, 24, 8], num_features=6, dims_bidir=[64], dim_dec=16, dim_matcher=16, conv_n=3,
                         conv_num_filters=2, num_phonemes=5, post_merge_activation="relu", maxout_pieces=1)
    rec = pkg.SpeechRecognizer(**dict(_kw(pkg, [16, 24, 8]), dim_matcher=16))
    assert rec.net["post_merge_dims"] == [16, 24, 8]
    assert rec._make_readout_config().num_layers == 3
    assert list(rec._make_readout_config().dims) == [16, 24, 8, 0]
    rec.set_initialization("/recognizer", weights_init=pkg.IsotropicGaussian(0.01), biases_init=pkg.Constant(0.0),
                           rec_weights_init=pkg.Orthogonal(), initial_states_init=pkg.IsotropicGaussian(0.001))
    shapes = RO.param_shapes(cfg)
    names = list(shapes)
    i = names.index(RO.PM + "/bias.b")
    assert names[i:i + 7] == [RO.PM + "/bias.b"] + [RO.linear_name(j) + leaf for j in range(3) for leaf in (".b", ".W")]
    assert shapes[RO.linear_name(0) + ".W"] == (16, 24) and shapes[RO.linear_name(2) + ".W"] == (8, 5)
    got = rec.initial_values(shapes, seed=1)
    want = RO.init_params(cfg, seed=1)
    assert list(got) == list(want)
    for k, v in want.items():
        assert_allclose(got[k], v.astype(np.float32), rtol=1e-6, atol=1e-9, err_msg=k)
    # prototype_speech.yaml's push onto the MLP
    rec.set_initialization(RO.PM + "/mlp", weights_init=pkg.Constant(0.5), biases_init=pkg.Constant(0.25))
    got = rec.initial_values(shapes, seed=1)
    for k, v in got.items():
        if k.startswith(RO.PM + "/mlp/"):
            assert (v == (0.5 if k.endswith(".W") else 0.25)).all(), k
    assert (got[RO.PM + "/bias.b"] == 0).all()
    # a depth-1 readout keeps the single-layer table and creates through the old entry points
    one = pkg.SpeechRecognizer(**_kw(pkg, [16]))
    assert one._make_readout_config() is None and one.net["post_merge_dims"] == [16]


def test_refusals_name_their_rule():
    pkg = package()
    with pytest.raises(NotImplementedError, match="post-merge MLP of 5 layers"):
        pkg.SpeechRecognizer(**_kw(pkg, [16] * 5))
    with pytest.raises(ValueError, match="multiple of 8"):
        pkg.SpeechRecognizer(**_kw(pkg, [16, 12]))
    with pytest.raises(ValueError, match="multiple of 8"):
        pkg.SpeechRecognizer(**_kw(pkg, [16, 0]))
    with pytest.raises(ValueError, match=r"Maxout\(2\).*one post-merge layer only"):
        pkg.SpeechRecognizer(**_kw(pkg, [16, 16], pkg.Maxout(2)))
    widest = pkg._lib.load().lvsr_readout_max_width()
    assert widest > 0 and widest % 8 == 0
    with pytest.raises(NotImplementedError, match="last post-merge width of %d" % (widest + 8)):
        pkg.SpeechRecognizer(**_kw(pkg, [16, widest + 8]))
    # accepted: Maxout(1) is the identity, the widest last width, every listed activation
    pkg.SpeechRecognizer(**_kw(pkg, [16, 16], pkg.Maxout(1)))
    pkg.SpeechRecognizer(**_kw(pkg, [16, 8, widest]))
    for act in (pkg.Tanh(), pkg.Rectifier(), pkg.Identity()):
        pkg.SpeechRecognizer(**_kw(pkg, [16, 16, 16, 16], act))
    # the bias-only readout stays refused
    with pytest.raises(NotImplementedError, match="readout without post_merge_dims"):
        pkg.SpeechRecognizer(**_kw(pkg, None))


def test_c_abi_refuses_before_device_work():
    """lvsr_model_create_readout checks the readout before it looks for a device: the same rules, with messages."""
    pkg = package()
    lib = pkg._lib.load()
    rec = pkg.SpeechRecognizer(**_kw(pkg, [16, 16]))
    cfg = rec._make_config()
    cfg.dim_matcher = 128

    def create(dims, pieces=1, act=pkg._lib.ACTIVATIONS["relu"]):
        cfg.maxout_pieces, cfg.post_merge_activation = pieces, act
        ro = pkg._lib.LvsrReadoutConfig()
        ro.num_layers = len(dims)
        for i, d in enumerate(dims[:pkg._lib.LVSR_MAX_READOUT]):
            ro.dims[i] = d
        h = ctypes.c_void_p()
        rc = lib.lvsr_model_create_readout(ctypes.byref(cfg), None, 1, ctypes.byref(ro), ctypes.byref(h))
        return rc, lib.lvsr_last_error().decode()

    widest = lib.lvsr_readout_max_width()
    for dims, pieces, act, msg in (([16] * 5, 1, "relu", "5 layers"), ([16, 20], 1, "relu", "multiple of 8"),
                                   ([8, 16], 1, "relu", "must equal post_merge_dim"),
                                   ([16, 16], 2, "maxout", "one post-merge layer only"),
                                   ([16, widest + 8], 1, "relu", "widest the readout kernels stage")):
        rc, err = create(dims, pieces, pkg._lib.ACTIVATIONS[act])
        assert rc != 0 and msg in err, (dims, err)


def test_config_keeps_dec_stack_last_and_version():
    pkg = package()
    fields = [f for f, _ in pkg._lib.LvsrConfig._fields_]
    assert fields[-1] == "dec_stack"
    with open(os.path.join(ROOT, "include", "lvsr_b200.h")) as f:
        header = f.read()
    body = re.search(r"typedef struct \{(.*?)\} lvsr_config;", header, re.S).group(1)
    assert re.findall(r"\b(\w+)(?:\[\w+\])?;", re.sub(r"/\*.*?\*/", "", body, flags=re.S))[-1] == "dec_stack"
    assert pkg._lib.load().lvsr_version() == 104
    ro = re.search(r"typedef struct \{([^}]*)\} lvsr_readout_config;", header, re.S).group(1)
    assert [f for f, _ in pkg._lib.LvsrReadoutConfig._fields_] == \
        re.findall(r"\b(\w+)(?:\[\w+\])?;", re.sub(r"/\*.*?\*/", "", ro, flags=re.S))


def _content_costs(cfg, params, batch):
    """The content model's cost matrix with the deep readout, from content_oracle's numpy decoder and RO.readout."""
    import content_oracle as CO
    x, m, labels, lm = batch
    r = CO.recognizer_cost(cfg, RO.shallow_params(cfg, params), x, m, labels, lm, return_all=True)
    logits = RO.readout(cfg, params, r["states"], r["weighted_averages"])
    return -np.take_along_axis(O.log_softmax(logits), labels[..., None], axis=-1)[..., 0] * lm


@pytest.mark.parametrize("dims,act,use_states", [([16, 24], "tanh", True), ([16, 8, 16], "relu", False)])
def test_content_mirror_and_its_gradient(dims, act, use_states):
    """The deep readout over content attention: RO.cost_and_grads on a content config runs content_oracle's loop with
    the deep readout; its costs equal content_oracle's decoder plus RO.readout, its gradients central differences."""
    pytest.importorskip("torch")
    import content_oracle as CO
    cfg = CO.make_config(num_features=6, dims_bidir=[8], dim_dec=8, dim_matcher=8, num_phonemes=5,
                         post_merge_dims=dims[:1], post_merge_activation=act, maxout_pieces=1,
                         use_states_for_readout=use_states)
    cfg["post_merge_dims"] = list(dims)
    deep = RO.init_params(small_cfg(dims, act, use_states), seed=2, scale=20.0)
    params = {}
    for k, v in CO.init_params(dict(cfg, post_merge_dims=dims[:1]), seed=2, scale=20.0).items():
        params[k] = deep[k] if k.startswith(RO.PM + "/") else v
    params.update((k, v) for k, v in deep.items() if k.startswith(RO.PM + "/mlp/"))
    batch = O.synthetic_batch(cfg, B=2, T=10, seed=4)
    cost, grads, costs = RO.cost_and_grads(cfg, params, *batch, return_costs=True)
    assert set(grads) == set(params)
    want = _content_costs(cfg, params, batch)
    assert_allclose(costs, want, rtol=1e-11, atol=1e-11)
    assert abs(cost - want.sum() / batch[2].shape[1]) < 1e-11
    # a deep readout changes the costs: the mirror does not fall back to the single-layer readout
    assert np.abs(want - CO.recognizer_cost(cfg, RO.shallow_params(cfg, params), *batch)).max() > 1e-3
    rng = np.random.RandomState(0)
    eps = 1e-6
    names = [RO.PM + "/bias.b", CO.CONT + "/energy_comp/linear.W", CO.CONT + "/state_trans/transform_states.W"] + \
        [RO.linear_name(j) + leaf for j in range(len(dims)) for leaf in (".W", ".b")]
    for name in names:
        assert grads[name].any(), name
        for _ in range(3):
            idx = tuple(rng.randint(n) for n in params[name].shape)
            plus, minus = dict(params), dict(params)
            plus[name], minus[name] = params[name].copy(), params[name].copy()
            plus[name][idx] += eps
            minus[name][idx] -= eps
            fd = (_content_costs(cfg, plus, batch).sum() - _content_costs(cfg, minus, batch).sum()) / (
                2 * eps * batch[2].shape[1])
            assert abs(fd - grads[name][idx]) <= 1e-6 * max(1.0, abs(fd)), (name, idx, fd, grads[name][idx])


def test_kink_screen_finds_every_rectifier_layer():
    """relu_kinks reports the pre-activations of h_0, h_1 and h_2 within eps of 0 on live rows, and nothing else;
    clear_kinks moves exactly those units' biases, the way that keeps the unit's other rows off the kink."""
    cfg = small_cfg([8, 8, 8], "relu", use_states=False)
    eps = 1e-5
    p = {k: np.zeros(v) for k, v in RO.param_shapes(cfg).items()}
    Wc = p[O._GEN + "/readout/merge/transform_weighted_averages.W"]
    for u in range(8):
        Wc[u, u] = 1.0                                              # z_0 = ctx[:8] + b
    p[RO.PM + "/bias.b"][:] = 0.5
    p[RO.linear_name(0) + ".W"][:] = np.eye(8)
    p[RO.linear_name(0) + ".b"][:] = -1.0                           # z_1 = h_0 - 1
    p[RO.linear_name(1) + ".W"][:] = np.eye(8)
    p[RO.linear_name(1) + ".b"][:] = 0.25                           # z_2 = relu(z_1) + 0.25
    p[RO.linear_name(1) + ".b"][5] = -2.0                           # z_2[5] = relu(z_1[5]) - 2
    ctx = np.ones((3, 2, 16))                                       # z_0 = 1.5, z_1 = 0.5 everywhere
    ctx[0, 1, 2] = -0.5 + 3e-6                                      # z_0[2] = 3e-6: h_0 kink
    ctx[2, 0, 4] = 0.5 - 4e-6                                       # z_1[4] = -4e-6: h_1 kink
    ctx[1, 1, 5] = 2.5 + 2e-6                                       # z_2[5] = 2e-6: h_2 kink
    ctx[1, 0, 6] = -0.5                                             # z_0[6] = 0 exactly, on a masked row
    ctx[2, 1, 2] = -0.5 - 2e-5                                      # z_0[2] = -2e-5: near, not within eps
    live = np.ones((3, 2), bool)
    live[1, 0] = False
    assert sorted(RO.relu_kinks(cfg, p, None, ctx, live, eps)) == [(0, 0, 1, 2), (1, 2, 0, 4), (2, 1, 1, 5)]
    assert (1, 1, 0, 6) not in RO.relu_kinks(cfg, p, None, ctx, None, eps) and \
        (0, 1, 0, 6) in RO.relu_kinks(cfg, p, None, ctx, None, eps)
    assert RO.relu_kinks(dict(cfg, post_merge_activation="tanh"), p, None, ctx, live, eps) == []
    cleared, moved = RO.clear_kinks(cfg, p, None, ctx, live, eps)
    # h_0 unit 2 has rows at 3e-6 and -2e-5: +3 eps leaves -2e-5 + 3e-5 = 1e-5 < 2 eps, -3 eps clears both
    assert [(j, u) for j, u, _ in moved] == [(0, 2), (1, 4), (2, 5)]
    assert_allclose([s for _, _, s in moved], [-3 * eps, 3 * eps, 3 * eps], rtol=1e-12)
    for k, v in p.items():
        changed = np.flatnonzero(np.asarray(cleared[k]).ravel() != v.ravel())
        want = {RO.PM + "/bias.b": [2], RO.linear_name(0) + ".b": [4], RO.linear_name(1) + ".b": [5]}.get(k, [])
        assert list(changed) == want, k
    assert RO.relu_kinks(cfg, cleared, None, ctx, live, eps) == []
    assert RO.clear_kinks(cfg, cleared, None, ctx, live, eps)[1] == []
