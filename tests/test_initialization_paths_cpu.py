"""Path-addressed initialisation (config['initialization'] beyond /recognizer, lvsr/main.py:223-231): the values
SpeechRecognizer.initial_values draws equal an independent restatement of the reference's walk -- schemes set on
the brick a path names and pushed down its subtree (B/bricks/base.py:713-729, B/bricks/interfaces.py:157-166),
the recognizer's recurrent push (lvsr/bricks/recognizer.py:362-373, lvsr/utils.py:1-14), then one RandomState
drawn in brick order (B/bricks/recurrent.py:568-580).  Host-only: the draws need no device."""
import sys
from collections import OrderedDict

import numpy as np
import pytest

from compat_helpers import COMPAT
from helpers import O, make_recognizer, package

NET = dict(num_features=6, dims_bidir=[4, 4], subsample=[1, 2], dim_dec=6, dim_matcher=8, conv_n=2,
           conv_num_filters=3, num_phonemes=5, post_merge_dims=[6], maxout_pieces=2, energy_normalizer="logistic")
ENERGY = "/recognizer/generator/att_trans/conv_att/energy_comp"


class _Brick(object):
    def __init__(self, path):
        self.path, self.children = path, []
        self.weights_init = self.biases_init = None
        # the GatedRecurrent bricks: the encoder's and the decoder's transition
        self.recurrent = path.endswith("/gatedrecurrent") or path.endswith("/transition")
        self.recurrent_weights_init = self.initial_states_init = None


def reference_walk(shapes, initialization, seed=1):
    """Restatement of lvsr/main.py:223-231 + Brick.initialize over a brick tree built from the parameter paths."""
    pkg = package()
    bricks = OrderedDict()

    def brick(path):
        if path not in bricks:
            bricks[path] = _Brick(path)
            parent = path.rsplit("/", 1)[0]
            if parent:
                brick(parent).children.append(bricks[path])
        return bricks[path]
    for name in shapes:
        brick(name.rsplit(".", 1)[0])
    root = bricks["/recognizer"]

    def push(b):                   # Initializable._push_initialization_config, then the children's pushes
        for c in b.children:
            if b.weights_init:
                c.weights_init = b.weights_init
            if b.biases_init:
                c.biases_init = b.biases_init
        for c in b.children:
            push(c)
    for path, attrs in sorted(initialization.items(), key=lambda kv: kv[0].count("/")):
        b, = [bricks[path]] if path in bricks else []
        for k, v in attrs.items():
            setattr(b, k, v)
        push(b)
        if b is root:              # SpeechRecognizer.push_initialization_config
            for x in bricks.values():
                if x.recurrent and getattr(root, "rec_weights_init", None):
                    x.weights_init = x.recurrent_weights_init = root.rec_weights_init
                if x.recurrent and getattr(root, "initial_states_init", None):
                    x.initial_states_init = root.initial_states_init
    rng = np.random.RandomState(seed)
    out = OrderedDict()
    for name, shape in shapes.items():
        b, leaf = bricks[name.rsplit(".", 1)[0]], name.rsplit(".", 1)[1]
        if leaf == "state_to_state":
            v = (b.recurrent_weights_init or b.weights_init).generate(rng, shape)
        elif leaf == "state_to_gates":
            d = shape[0]
            v = np.hstack([b.weights_init.generate(rng, (d, d)), b.weights_init.generate(rng, (d, d))])
        elif leaf == "initial_state":
            v = (b.initial_states_init or pkg.Constant(0.0)).generate(rng, shape)
        elif leaf == "b":
            v = b.biases_init.generate(rng, shape)
        else:
            v = b.weights_init.generate(rng, shape)
        out[name] = np.asarray(v, np.float32).reshape(shape)
    return out


def _root(pkg):
    return {"/recognizer": dict(weights_init=pkg.IsotropicGaussian(0.1), biases_init=pkg.Constant(0.0),
                                rec_weights_init=pkg.Orthogonal(), initial_states_init=pkg.IsotropicGaussian(0.001))}


def _draw(initialization, seed=1):
    cfg = O.make_config(**NET)
    rec = make_recognizer(cfg)
    for path, schemes in initialization.items():
        rec.set_initialization(path, **schemes)
    shapes = O.param_shapes(cfg)
    return rec.initial_values(shapes, seed), reference_walk(shapes, initialization, seed)


def _same(got, want):
    assert list(got) == list(want)
    for k in want:
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)


def test_constant_override_changes_that_brick_and_the_stream_after_it():
    """exp/wsj/configs/wsj_jan_bhd04.yaml: energy_comp's weights Constant 0.  A Constant draws nothing: the parameters
    drawn before energy_comp keep the values of the run without the override, the ones after it take the draws the
    Gaussian of energy_comp would have consumed."""
    pkg = package()
    init = _root(pkg)
    base, _ = _draw(init)
    init[ENERGY] = dict(weights_init=pkg.Constant(0.0))
    got, want = _draw(init)
    _same(got, want)
    assert not got[ENERGY + "/linear.W"].any() and base[ENERGY + "/linear.W"].any()
    assert not got[ENERGY + "/linear.b"].any()
    names = list(got)
    at = names.index(ENERGY + "/linear.W")
    for k in names[:at]:
        np.testing.assert_array_equal(got[k], base[k], err_msg=k)
    # handler.W is the next draw: it starts where energy_comp's weights started in the run without the override
    n = base[ENERGY + "/linear.W"].size
    handler = "/recognizer/generator/att_trans/conv_att/handler.W"
    assert names[at + 1] == handler
    np.testing.assert_array_equal(got[handler].ravel()[:n], base[ENERGY + "/linear.W"].ravel())


def test_uniform_override_shifts_the_later_draws_of_the_one_stream():
    """A Uniform over the attention brick draws from the same RandomState as everything else: its parameters lie in
    the Uniform's support and every parameter drawn after them moves with the stream."""
    pkg = package()
    init = _root(pkg)
    base, _ = _draw(init)
    att = "/recognizer/generator/att_trans/conv_att"
    init[att] = dict(weights_init=pkg.Uniform(width=0.1), biases_init=pkg.Constant(0.25))
    got, want = _draw(init)
    _same(got, want)
    names = list(got)
    first = min(i for i, k in enumerate(names) if k.startswith(att + "/"))
    for k in names[:first]:
        np.testing.assert_array_equal(got[k], base[k], err_msg=k)
    for k in names[first:]:
        if k.startswith(att + "/"):
            v = got[k]
            if k.endswith(".b"):
                assert (v == 0.25).all(), k
            else:
                assert np.abs(v).max() <= 0.05 and np.abs(v).max() > 0.02, k
        elif not k.endswith(".b"):
            assert not np.array_equal(got[k], base[k]), k          # drawn later from the same stream


def test_override_over_a_recurrent_brick_takes_its_gate_matrices():
    """A path over an encoder direction pushes weights_init into its GatedRecurrent: the gate matrices follow the
    path, state_to_state keeps the recognizer's rec_weights_init, the initial state its initial_states_init.  Without
    a rec_weights_init the path decides state_to_state too."""
    pkg = package()
    fwd = "/recognizer/encoder/bidir0/forward"
    for with_rec in (True, False):
        init = _root(pkg)
        if not with_rec:
            del init["/recognizer"]["rec_weights_init"]
        init[fwd] = dict(weights_init=pkg.Uniform(width=0.1))
        got, want = _draw(init)
        _same(got, want)
        assert np.abs(got[fwd + "/gatedrecurrent.state_to_gates"]).max() <= 0.05
        assert (np.abs(got[fwd + "/gatedrecurrent.state_to_state"]).max() <= 0.05) == (not with_rec)
        assert np.abs(got[fwd + "/fork/fork_inputs.W"]).max() <= 0.05


def test_deeper_path_wins_over_a_shallower_one():
    """Paths are pushed by depth (lvsr/main.py:225-227): the deeper one holds for its subtree, whatever the order of
    the configuration's entries."""
    pkg = package()
    init = OrderedDict()
    init[ENERGY] = dict(weights_init=pkg.Constant(0.5))
    init["/recognizer/generator"] = dict(weights_init=pkg.Constant(-0.5))
    init.update(_root(pkg))
    got, want = _draw(init)
    _same(got, want)
    assert (got[ENERGY + "/linear.W"] == 0.5).all()
    assert (got["/recognizer/generator/att_trans/conv_att/handler.W"] == -0.5).all()


def test_unknown_path_and_scheme_are_refused():
    """A path that names no brick fails as the reference's `brick, = Selector(recognizer).select(path).bricks` does;
    a brick below /recognizer takes weights_init and biases_init only."""
    pkg = package()
    cfg = O.make_config(**NET)
    rec = make_recognizer(cfg)
    rec.set_initialization("/recognizer/generator/att_trans/conv_att/energy_comb", weights_init=pkg.Constant(0.0))
    with pytest.raises(ValueError, match="no brick"):
        rec.initial_values(O.param_shapes(cfg))
    with pytest.raises(ValueError):
        reference_walk(O.param_shapes(cfg), {"/recognizer/nope": dict(weights_init=pkg.Constant(0.0))})
    with pytest.raises(TypeError):
        make_recognizer(cfg).set_initialization(ENERGY, rec_weights_init=pkg.Orthogonal())


def test_uniform_of_a_yaml_mapping_loads_and_draws_within_its_width(tmp_path):
    """`!!python/object:blocks.initialization.Uniform {width: 0.1}` (exp/wsj/configs/wsj_jan_bhd04.yaml) builds the
    object without calling __init__; it still draws from U(-0.05, 0.05)."""
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as C
    path = tmp_path / "init.yaml"
    path.write_text("initialization:\n"
                    "    /recognizer:\n"
                    "        weights_init:\n"
                    "          !!python/object:blocks.initialization.Uniform {width: 0.1}\n"
                    "    %s:\n"
                    "        weights_init:\n"
                    "          !!python/object/apply:blocks.initialization.Constant [0.]\n" % ENERGY)
    cfg = C.Configuration(str(path), None, [])
    u = cfg["initialization"]["/recognizer"]["weights_init"]
    assert isinstance(u, package().Uniform)
    v = u.generate(np.random.RandomState(3), (4000,))
    assert np.abs(v).max() <= 0.05 and v.min() < -0.049 and v.max() > 0.049
