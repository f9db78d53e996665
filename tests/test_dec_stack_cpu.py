"""The stacked decoder (net.dec_stack: 2) without a GPU: the float64 stack oracle, its parameter table, the
configuration plumbing and the refusal to train."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest
from numpy.testing import assert_allclose

from oracle import lvsr_oracle as O
import content_oracle as CO
import stack_oracle as SO
import test_gpu_widths as W
from compat_helpers import COMPAT, write_experiment
from helpers import ROOT, package

TINY = dict(num_features=6, dims_bidir=[16, 16], subsample=[1, 2], dim_dec=16, dim_matcher=24, conv_n=3,
            conv_num_filters=4, num_phonemes=10, post_merge_dims=[16], maxout_pieces=2)
WINDOW = dict(type="window_around_mean", before=3, after=3, initial_begin=0, initial_end=100, min_speed=0,
              max_speed=0)


def _pair(attention_type, **kw):
    """(single-layer config and oracle module, stack config) of the same model."""
    if attention_type == "content":
        return CO.make_config(**dict(TINY, **kw)), CO, SO.make_config("content", **dict(TINY, **kw))
    return O.make_config(**dict(TINY, **kw)), O, SO.make_config(**dict(TINY, **kw))


@pytest.mark.parametrize("attention_type,extra", [
    ("content_and_conv", {}),
    ("content_and_conv", dict(prior=WINDOW, energy_normalizer="logistic", embed_outputs=False)),
    ("content", {}),
])
def test_zero_upper_layer_is_the_single_layer_model(attention_type, extra):
    """Layer 1 and every "#1" input zero, initial state included: layer 1's state stays 0 (tanh(0) = 0 blended with
    0), the attention and the readout see only s0, and layer 0 with its costs is the single-layer oracle's."""
    cfg1, M1, cfg2 = _pair(attention_type, **extra)
    single = M1.init_params(cfg1, seed=3, scale=10.0)
    stack = SO.from_single(cfg2, single)
    x, m, labels, lm = O.synthetic_batch(cfg1, B=3, T=20, seed=5)
    want = M1.recognizer_cost(cfg1, single, x, m, labels, lm, return_all=True)
    got = SO.recognizer_cost(cfg2, stack, x, m, labels, lm, return_all=True)
    C = cfg1["dim_dec"]
    assert got["states"].shape == want["states"].shape[:2] + (2 * C,)
    assert not np.any(got["states"][..., C:])
    for key in ("costs", "weights", "energies", "weighted_averages"):
        assert_allclose(got[key], want[key], rtol=0, atol=1e-12, err_msg=key)
    assert_allclose(got["states"][..., :C], want["states"], rtol=0, atol=1e-12)
    assert SO.beam_search(cfg2, stack, x[:, 0], 3, max_length=6) == M1.beam_search(cfg1, single, x[:, 0], 3,
                                                                                    max_length=6)


WIDTHS = [(c, True) for c in W.CASES] + [("ragged_k", False), ("odd_c", False)]


@pytest.mark.parametrize("case,states_readout", WIDTHS,
                         ids=[c + ("" if s else "-no_states_readout") for c, s in WIDTHS])
def test_zero_upper_layer_at_every_width(case, states_readout):
    """The same at the widths of test_gpu_widths.CASES (C = 8 to 512, E = 256 and 512, one-hot feedback, Maxout(3),
    Tanh, Rectifier, Identity, V = 2 to 128, content attention) and without the states in the readout, on the
    teacher-forced decoder alone."""
    net, prior = W.CASES[case]
    kw = dict(W.COMMON, **net, use_states_for_readout=states_readout)
    if case.startswith("content"):
        cfg1, M1, cfg2 = CO.make_config(**kw), CO, SO.make_config("content", **kw)
    else:
        cfg1, M1, cfg2 = O.make_config(prior=prior, **kw), O, SO.make_config(prior=prior, **kw)
    single = M1.init_params(cfg1, seed=3, scale=10.0)
    stack = SO.from_single(cfg2, single)
    assert any("readout/merge/transform_states#1" in k for k in stack) == states_readout
    att, attm, labels, lm = W._inputs(cfg1, 3, 14, 6, seed=4)
    want = M1.cost_matrix(cfg1, single, att, attm, labels, lm, return_all=True)
    got = SO.cost_matrix(cfg2, stack, att, attm, labels, lm, return_all=True)
    C = cfg1["dim_dec"]
    assert got["states"].shape == want["states"].shape[:2] + (2 * C,)
    assert not np.any(got["states"][..., C:])
    for key in ("costs", "weights", "energies", "weighted_averages"):
        assert_allclose(got[key], want[key], rtol=0, atol=1e-12, err_msg=key)
    assert_allclose(got["states"][..., :C], want["states"], rtol=0, atol=1e-12)


def test_transition_is_blocks_recurrent_stack_with_skip_connections():
    """Blocks' TestRecurrentStack.do_many_steps (libs/blocks/tests/bricks/test_recurrent.py:325-417) with
    skip_connections=True, restated for GatedRecurrent layers: 24 steps of 4 rows, the same inputs (permutations of
    0.1 * range(12)) to every layer, the last 12 steps of row 3 masked, every weight 2; each layer above the bottom
    adds the fork of the new state of the layer below to its own inputs."""
    import itertools
    depth, D = 2, 3
    x_val = 0.1 * np.asarray(list(itertools.islice(itertools.permutations(range(12)), 0, 24)), dtype=np.float64)
    x_val = np.ones((24, 4, 12)) * x_val[:, None, :]
    mask_val = np.ones((24, 4))
    mask_val[12:24, 3] = 0
    W_state2x = 2 * np.ones((D, 3 * D))          # fork of a layer's state into the next layer's [inputs | gates]
    W_s2g, W_s2s = 2 * np.ones((D, 2 * D)), 2 * np.ones((D, D))
    h_val = np.zeros((depth, 25, 4, D))

    def sigmoid(v):
        return 1. / (1. + np.exp(-v))

    for i in range(1, 25):
        below = None
        for d in range(depth):
            h_v = h_val[d][i - 1]
            inp, gate = x_val[i - 1][:, :D], x_val[i - 1][:, D:3 * D]
            if d > 0:
                fork = below.dot(W_state2x)
                inp, gate = inp + fork[:, :D], gate + fork[:, D:]
            g = sigmoid(h_v.dot(W_s2g) + gate)
            z, r = g[:, :D], g[:, D:]
            h_v1 = np.tanh((h_v * r).dot(W_s2s) + inp) * z + h_v * (1 - z)
            h_v = mask_val[i - 1, :, None] * h_v1 + (1 - mask_val[i - 1, :, None]) * h_v
            h_val[d][i] = h_v
            below = h_v

    layers = [dict(state_to_state=W_s2s, state_to_gates=W_s2g)] * depth
    forks = [dict(inputs=W_state2x[:, :D], gate_inputs=W_state2x[:, D:])]
    states = [np.zeros((4, D))] * depth
    for i in range(24):
        inputs = [(x_val[i][:, :D], x_val[i][:, D:3 * D])] * depth
        states = SO.recurrent_stack_step(layers, forks, states, inputs, mask_val[i])
        for d in range(depth):
            assert_allclose(states[d], h_val[d][i + 1], rtol=1e-13, atol=0)
    assert np.all(h_val[:, 13:, 3] == h_val[:, 12:13, 3])         # masked steps keep the state


def test_wide_state_products_are_the_sums_of_the_reference():
    """take_glimpses and the readout on [s0 | s1] with wide_params equal the reference's sum of one Linear per state
    (state_trans Parallel, lvsr/bricks/attention.py:103-106; readout Merge, lvsr/bricks/recognizer.py:298-301)."""
    cfg = SO.make_config(**TINY)
    p = SO.init_params(cfg, seed=2, scale=10.0)
    wide = SO.wide_params(cfg, p)
    rng = np.random.RandomState(0)
    C, B = cfg["dim_dec"], 3
    s = rng.normal(size=(B, 2 * C))
    wa = rng.normal(size=(B, O.dim_encoded(cfg)))
    g = O._GEN + "/readout/merge/"
    r = wa.dot(p[g + "transform_weighted_averages.W"]) + s[:, :C].dot(p[g + "transform_states.W"]) + \
        s[:, C:].dot(p[g + "transform_states#1.W"]) + p[O._GEN + "/readout/post_merge/bias.b"]
    r = O.maxout(r, 2).dot(p[O._GEN + "/readout/post_merge/mlp/linear_0.W"]) + p[O._GEN + "/readout/post_merge/mlp/linear_0.b"]
    assert_allclose(O.readout(cfg, wide, s, wa), r, rtol=1e-13, atol=1e-15)
    a = O._ATT + "/state_trans/"
    q = s[:, :C].dot(p[a + "transform_states.W"]) + s[:, C:].dot(p[a + "transform_states#1.W"])
    assert_allclose(s.dot(wide[a + "transform_states.W"]), q, rtol=1e-13, atol=1e-15)


# wsj_jan_wsj13v2.yaml: wsj_jan_new.yaml (one-of-N feedback, dim_dec 256, dim_matcher 512, conv_n 100, 10 filters,
# Maxout(2) post-merge of 256) with 3 BiGRU layers of 256, subsampling [1, 1, 2] and dec_stack 2
WSJ13V2 = dict(num_features=123, dims_bidir=[256, 256, 256], subsample=[1, 1, 2], dim_dec=256, dim_matcher=512,
               conv_n=100, conv_num_filters=10, num_phonemes=32, post_merge_dims=[256], maxout_pieces=2,
               embed_outputs=False, prior=dict(type="window_around_mean", before=150, after=150, initial_begin=0,
                                               initial_end=100, min_speed=3, max_speed=5.5))

_G, _T = "/recognizer/generator", "/recognizer/generator/att_trans"
WSJ13V2_DECODER = [            # after the encoder's 42 parameters, in Blocks' initialisation order
    (_G + "/readout/merge/transform_states.W", (256, 256)),
    (_G + "/readout/merge/transform_states#1.W", (256, 256)),
    (_G + "/readout/merge/transform_weighted_averages.W", (512, 256)),
    (_G + "/readout/post_merge/bias.b", (256,)),
    (_G + "/readout/post_merge/mlp/linear_0.b", (32,)),
    (_G + "/readout/post_merge/mlp/linear_0.W", (128, 32)),
    (_G + "/fork/fork_inputs.b", (256,)),
    (_G + "/fork/fork_inputs.W", (33, 256)),
    (_G + "/fork/fork_gate_inputs.b", (512,)),
    (_G + "/fork/fork_gate_inputs.W", (33, 512)),
    (_G + "/fork/fork_inputs#1.b", (256,)),
    (_G + "/fork/fork_inputs#1.W", (33, 256)),
    (_G + "/fork/fork_gate_inputs#1.b", (512,)),
    (_G + "/fork/fork_gate_inputs#1.W", (33, 512)),
    (_T + "/recurrentstack/transition_0#0.state_to_state", (256, 256)),
    (_T + "/recurrentstack/transition_0#0.state_to_gates", (256, 512)),
    (_T + "/recurrentstack/transition_0#0.initial_state", (256,)),
    (_T + "/recurrentstack/transition_1#1.state_to_state", (256, 256)),
    (_T + "/recurrentstack/transition_1#1.state_to_gates", (256, 512)),
    (_T + "/recurrentstack/transition_1#1.initial_state", (256,)),
    (_T + "/recurrentstack/fork_1/fork_inputs.W", (256, 256)),
    (_T + "/recurrentstack/fork_1/fork_gate_inputs.W", (256, 512)),
    (_T + "/conv_att/state_trans/transform_states.W", (256, 512)),
    (_T + "/conv_att/state_trans/transform_states#1.W", (256, 512)),
    (_T + "/conv_att/preprocess.b", (512,)),
    (_T + "/conv_att/preprocess.W", (512, 512)),
    (_T + "/conv_att/energy_comp/linear.W", (512, 1)),
    (_T + "/conv_att/handler.W", (10, 512)),
    (_T + "/conv_att/conv1d.filters", (10, 201)),
    (_T + "/distribute/fork_inputs.W", (512, 256)),
    (_T + "/distribute/fork_gate_inputs.W", (512, 512)),
    (_T + "/distribute/fork_inputs#1.W", (512, 256)),
    (_T + "/distribute/fork_gate_inputs#1.W", (512, 512)),
]


def test_wsj13v2_parameter_table():
    """The Blocks names of the stack: RecurrentStack sits in att_trans as "recurrentstack" and renames its layers
    "transition_<l>#<l>" (recurrent.py:819-820); fork_1 is a Fork over layer 1's own sequence names without bias
    (recurrent.py:828-831, Linear(use_bias=not skip_connections)); every brick fed by the states or the sequences
    gets a "#1" child (Parallel/Fork name children <prefix>_<input name>)."""
    shapes = SO.param_shapes(SO.make_config(**WSJ13V2))
    items = list(shapes.items())
    assert len(items) == 42 + len(WSJ13V2_DECODER)
    assert all(k.startswith("/recognizer/encoder/") for k, _ in items[:42])
    assert items[42:] == WSJ13V2_DECODER


def test_initialization_walks_the_stack_in_brick_order():
    """initialize() on the stack's table under the WSJ schemes draws what the oracle's init_params draws: one
    RandomState in brick order (both layers, then fork_1), rec_weights_init and initial_states_init on both layers
    (lvsr/bricks/recognizer.py:363-373 pushes them onto every BaseRecurrent), weights_init on fork_1."""
    pkg = package()
    cfg = SO.make_config(**TINY)
    rec = pkg.SpeechRecognizer(input_dims={"recordings": 6}, input_num_chars={}, eos_label=9, num_phonemes=10,
                               dim_dec=16, dims_bidir=[16, 16], subsample=[1, 2], conv_n=3, conv_num_filters=4,
                               dim_matcher=24, post_merge_dims=[16], post_merge_activation=pkg.Maxout(2), dec_stack=2)
    rec.set_initialization("/recognizer", weights_init=pkg.IsotropicGaussian(0.01), biases_init=pkg.Constant(0.0),
                           rec_weights_init=pkg.Orthogonal(), initial_states_init=pkg.IsotropicGaussian(0.001))
    got = rec.initial_values(SO.param_shapes(cfg), seed=1)
    want = SO.init_params(cfg, seed=1)
    assert list(got) == list(want)
    for k, v in want.items():
        assert_allclose(got[k], v.astype(np.float32), rtol=1e-6, atol=1e-9, err_msg=k)


def test_config_plumbing():
    """dec_stack reaches lvsr_config as its last field (zero-filled by older callers, which the library reads as 1);
    1 and 2 are accepted, anything else is refused."""
    pkg = package()
    fields = [f for f, _ in pkg._lib.LvsrConfig._fields_]
    assert fields[-1] == "dec_stack" and pkg._lib.LvsrConfig().dec_stack == 0
    with open(os.path.join(ROOT, "include", "lvsr_b200.h")) as f:
        header = f.read()
    body = re.search(r"typedef struct \{(.*?)\} lvsr_config;", header, re.S).group(1)
    assert re.findall(r"\b(\w+)(?:\[\w+\])?;", re.sub(r"/\*.*?\*/", "", body, flags=re.S))[-1] == "dec_stack"
    assert ctypes.sizeof(pkg._lib.LvsrConfig) % 8 == 0
    kw = dict(input_dims={"recordings": 6}, input_num_chars={}, eos_label=9, num_phonemes=10, dim_dec=16,
              dims_bidir=[16], conv_n=3, post_merge_dims=[16], post_merge_activation=pkg.Maxout(2))
    for stack in (1, 2):
        rec = pkg.SpeechRecognizer(dec_stack=stack, **kw)
        assert rec._make_config().dec_stack == stack and rec.dim_state == 16 * stack
    for bad in (0, 3):
        with pytest.raises(NotImplementedError, match="dec_stack"):
            pkg.SpeechRecognizer(dec_stack=bad, **kw)


def test_training_a_stack_is_refused(tmp_path):
    """GradientDescent and compat's train refuse dec_stack 2 before any device work."""
    pkg = package()
    rec = pkg.SpeechRecognizer(input_dims={"recordings": 6}, input_num_chars={}, eos_label=9, num_phonemes=10,
                               dim_dec=16, dims_bidir=[16], conv_n=3, post_merge_dims=[16],
                               post_merge_activation=pkg.Maxout(2), dec_stack=2)
    with pytest.raises(NotImplementedError, match="dec_stack=2"):
        pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as LC
    import lvsr.main as LM
    exp = write_experiment(tmp_path)
    cfg = LC.Configuration(exp["base"], "$LVSR/lvsr/configs/schema.yaml", [("net.dec_stack", "2")])
    with pytest.raises(NotImplementedError, match="dec_stack=2"):
        LM.train(cfg, os.path.join(str(tmp_path), "model"))
