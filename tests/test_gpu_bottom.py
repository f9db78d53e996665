"""The bottom MLP (net.bottom.dims) on the GPU against the float64 bottom oracle (tests/bottom_oracle.py): the parameter
table and the refusals of lvsr_model_create_bottom, the encoder output and the cost matrix at every operand path of its
GEMMs (fp16 head/tail at 128 features, 3xTF32 at 40, FFMA tiles at 123 features or a width that is not a multiple of
128) for both activations, one and two layers, both attention types and dec_stack 2; generation, beam search one
utterance at a time and in lock-step, LM-fused costs, analyze and validation_statistics; the training step's gradients,
two optimizer steps, one step under adaptive noise and the independence from the padded frames' values; the checkpoint
round trip and a compat train -> search run.

Element-wise bounds are test_gpu_attention_plans.py's for the decoder (it decodes the GPU's own encoder output) and
1e-4 per element (floor 0.1 of the largest magnitude) for the encoder output; gradients are held to check_grads' 1e-4.
Rectifier cases assert that no pre-activation of a live frame lies within 1e-5 of 0, where a float32 value could take
the other side of the kink."""
import ctypes
import os
import sys
from collections import OrderedDict

import numpy as np
import pytest

import bottom_oracle as BO
import content_oracle as CO
import lm_oracle as LO
import stack_oracle as SO
from compat_helpers import COMPAT, write_experiment
from helpers import O, elementwise_err, f32, package, rel_err
from helpers import bottom_params as _params, bottom_recognizer as _recognizer
from oracle import lvsr_oracle_grad as G
from test_gpu_attention_plans import TOL, _compare
from test_gpu_widths import _same_up_to_near_ties

pytestmark = pytest.mark.gpu

SMALL = dict(num_features=40, dims_bidir=[128], subsample=[1], dim_dec=128, dim_matcher=256, conv_n=8,
             conv_num_filters=10, num_phonemes=32, post_merge_dims=[128], maxout_pieces=2)
PYRAMID = dict(SMALL, dims_bidir=[128, 128], subsample=[1, 2])
MEDIAN = dict(type="window_around_median", before=5, after=7)
_RO = "/recognizer/generator/readout/post_merge/mlp/linear_0"


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _config(arch, dims, activation, attention_type="content_and_conv", dec_stack=1, **extra):
    kw = dict(arch, **extra)
    if dec_stack == 2:
        base = SO.make_config(attention_type, **kw)
    else:
        base = CO.make_config(**kw) if attention_type == "content" else O.make_config(**kw)
    return BO.make_config(base, dims, activation)




def test_parameter_table_and_refusals():
    """The library's table is the oracle's; NULL and zero layers give the table without a bottom; every depth, width
    and activation outside lvsr_bottom_config's ranges is refused at creation with its reason."""
    _torch()
    pkg = package()
    lib = pkg._lib.load()
    cfg = _config(dict(SMALL, num_features=123), [256, 250], "relu")
    rec = _recognizer(cfg)
    assert list(rec.parameter_shapes().items()) == list(BO.param_shapes(cfg).items())
    plain = pkg.SpeechRecognizer(input_dims={"recordings": 123}, input_num_chars={}, eos_label=31, num_phonemes=32,
                                 dim_dec=128, dims_bidir=[128], conv_n=8, conv_num_filters=10, dim_matcher=256,
                                 post_merge_dims=[128], post_merge_activation=pkg.Maxout(2))
    c = plain._make_config()

    def create(bottom):
        h = ctypes.c_void_p()
        rc = lib.lvsr_model_create_bottom(ctypes.byref(c), None if bottom is None else ctypes.byref(bottom),
                                          ctypes.byref(h))
        if rc != 0:
            return lib.lvsr_last_error().decode()
        try:
            return [lib.lvsr_model_param_name(h, i).decode() for i in range(lib.lvsr_model_num_params(h))]
        finally:
            lib.lvsr_model_destroy(h)

    def bottom(n, dims, act):
        b = pkg._lib.LvsrBottomConfig()
        b.num_layers = n
        for i, d in enumerate(dims):
            b.dims[i] = d
        b.activation = act
        return b

    assert create(None) == create(bottom(0, [], 0)) == list(plain.parameter_shapes())
    assert "5 layers" in create(bottom(5, [8, 8, 8, 8], 1))
    assert "-1 layers" in create(bottom(-1, [], 1))
    assert "width 0 of layer 1" in create(bottom(2, [8, 0], 1))
    assert "width 4097 of layer 0" in create(bottom(1, [4097], 2))
    assert isinstance(create(bottom(1, [4096], 2)), list)
    for act in (0, 3, 7):
        assert "activation %d" % act in create(bottom(1, [8], act))


# name, arch, dims, activation, extra: both operand kinds of the bottom's own GEMM and of encoder layer 0 after it
COST_CASES = [
    ("f40_relu256_tf32", SMALL, [256], "relu", {}),
    ("f128_tanh256_f16", dict(SMALL, num_features=128), [256], "tanh", {}),
    ("f123_relu100_ffma", dict(SMALL, num_features=123), [100], "relu", {}),
    ("f40_relu256_250_ragged", PYRAMID, [256, 250], "relu", {}),
    ("f128_tanh250_100_content", dict(SMALL, num_features=128), [250, 100], "tanh", dict(attention_type="content")),
    ("f40_relu256_stack", SMALL, [256], "relu", dict(dec_stack=2, prior=MEDIAN)),
    ("f123_tanh256_stack_content", dict(SMALL, num_features=123), [256], "tanh",
     dict(dec_stack=2, attention_type="content")),
]


@pytest.mark.parametrize("case,arch,dims,activation,extra", COST_CASES, ids=[c[0] for c in COST_CASES])
def test_encoder_and_cost_matrix_match_oracle(case, arch, dims, activation, extra):
    """The encoder output against the whole float64 encoder with its bottom; the cost matrix (costs, weights, energies,
    states, glimpses) decoded from it; the host entry point (bottom + encoder + decoder) against the whole model."""
    torch = _torch()
    cfg = _config(arch, dims, activation, **extra)
    params = _params(cfg, seed=3)
    rec = _recognizer(cfg, params)
    x, m, labels, lm = O.synthetic_batch(cfg, B=5, T=48, seed=5)
    att, attm = rec.encode(x, m)
    o_att, o_attm = BO.encoder(cfg, params, x, m)
    err = elementwise_err(att.cpu().numpy(), o_att)
    print("ERR encoder", case, "%.2e" % err)
    assert err <= 1e-4, (case, err)
    assert np.array_equal(attm.cpu().numpy(), o_attm)
    att64, attm64 = f32(att.cpu().numpy()), attm.cpu().numpy().astype(np.float64)
    got = rec.cost_matrix(labels, lm, att, attm, return_all=True)
    torch.cuda.synchronize()
    M = BO._module(cfg)
    want = M.cost_matrix(BO.inner(cfg), params, att64, attm64, labels, lm, return_all=True)
    _compare(got, want, cfg.get("attention_type") == "content", case)
    assert rel_err(rec.cost(x, m, labels, lm), BO.recognizer_cost(cfg, params, x, m, labels, lm)) < 1e-4


@pytest.mark.parametrize("attention_type,dec_stack", [("content_and_conv", 1), ("content", 1), ("content_and_conv", 2)])
def test_greedy_and_sampled_generation(attention_type, dec_stack):
    """generate(sample=False) emits the oracle's arg-max tokens from the GPU's encoding; sample() draws from a device
    stream, so its costs are checked against the oracle's teacher-forced costs of the drawn tokens."""
    _torch()
    cfg = _config(SMALL, [256], "relu", attention_type=attention_type, dec_stack=dec_stack)
    params = _params(cfg, seed=7, gain=3.0)
    rec = _recognizer(cfg, params)
    x, m, _, _ = O.synthetic_batch(cfg, B=5, T=36, seed=9)
    att, attm = rec.encode(x, m)
    att64, attm64 = f32(att.cpu().numpy()), attm.cpu().numpy().astype(np.float64)
    n = 12
    got = rec.generate(x, m, n_steps=n, sample=False)
    M = BO._module(cfg)
    outs, costs, _ = M.generate_greedy(BO.inner(cfg), params, att64, attm64, n)
    assert np.array_equal(got["outputs"], outs)
    assert elementwise_err(got["costs"], costs) <= TOL["costs"]
    drawn = rec.generate(x, m, n_steps=n, sample=True, seed=4)
    want = M.cost_matrix(BO.inner(cfg), params, att64, attm64, drawn["outputs"].astype(np.int64))
    assert elementwise_err(drawn["costs"], want) <= TOL["costs"]
    assert rec.sample({"recordings": x[:, 0]}, n_steps=4, seed=1).shape == (4, 1)


@pytest.mark.parametrize("beam", [1, 10])
@pytest.mark.parametrize("dec_stack", [1, 2])
def test_beam_search_matches_oracle(beam, dec_stack):
    """Every finished hypothesis with its cost against the whole float64 model, one utterance at a time and in
    search_many's lock-step; token for token."""
    _torch()
    scale = 2.0
    cfg = _config(SMALL, [256, 250], "tanh", dec_stack=dec_stack, prior=MEDIAN, max_decoded_length_scale=scale)
    params = _params(cfg, seed=11, gain=4.0, eos_bias=6.0)
    rec = _recognizer(cfg, params)
    rec.init_beam_search(beam)
    rng = np.random.RandomState(13)
    utts = [rng.normal(size=(T, cfg["num_features"])) for T in (40, 27, 33, 46)]
    many = rec.beam_search_many([{"recordings": u.astype(np.float32)} for u in utts])
    found = 0
    for u, g in zip(utts, many):
        try:
            want = BO.beam_search(cfg, params, u, beam)
        except O.CandidateNotFoundError:
            assert g is None
            continue
        one = rec.beam_search({"recordings": u.astype(np.float32)})
        for res in (one, g):
            if beam == 1:
                assert res[0] == want[0]
                assert elementwise_err(res[1], want[1]) <= 1e-5
            else:
                _same_up_to_near_ties(res, want)
        found += 1
    assert found >= 3


@pytest.fixture(scope="module")
def lm_file(tmp_path_factory):
    V = SMALL["num_phonemes"]
    S, start, arcs = LO.char_ngram(V, seed=7, n_tri=60, dup=6, dead=2)
    path = str(tmp_path_factory.mktemp("lm") / "lm.fst")
    cmap = LO.to_file(path, V, S, start, arcs, seed=2)
    return path, cmap, LO.from_tables(package().lm.load(path, cmap, V))


def test_lm_fused_teacher_forcing(lm_file):
    """cost() with an FST language model: the fused costs of the oracle on the bottom's encoding."""
    _torch()
    path, cmap, fst = lm_file
    cfg = _config(SMALL, [256], "relu")
    params = _params(cfg, seed=4)
    rec = _recognizer(cfg, params, lm=dict(path=path, no_transition_cost=20.0, weight=0.5), cmap=cmap)
    x, m, labels, lmask = O.synthetic_batch(cfg, B=3, T=40, seed=5)
    att, attm = BO.encoder(cfg, params, x, m)
    want = LO.cost_matrix(BO.inner(cfg), params, fst, rec.lm, att, attm, labels, lmask, oracle=O)
    assert np.allclose(rec.cost(x, m, labels, lmask), want, rtol=1e-4, atol=1e-4)


def test_analyze_and_validation_statistics():
    _torch()
    cfg = _config(SMALL, [256, 100], "relu")
    params = _params(cfg, seed=5)
    rec = _recognizer(cfg, params)
    x, m, labels, lm = O.synthetic_batch(cfg, B=4, T=40, seed=6)
    costs, weights, energies = rec.analyze({"recordings": x[:, 0]}, labels[:, 0])
    wc, ww, we = O.analyze(BO.inner(cfg), params, BO.bottom(cfg, params, x[:, 0]), labels[:, 0])
    assert rel_err(costs, wc) < 1e-4 and rel_err(weights, ww) < 1e-4 and rel_err(energies, we) < 1e-4
    stats = rec.validation_statistics(x, m, labels, lm)
    want = BO.recognizer_cost(cfg, params, x, m, labels, lm)
    assert abs(stats["cost"] - want.sum()) <= 1e-4 * abs(want.sum())
    assert stats["num_labels"] == lm.sum() and stats["batch_size"] == 4


# ---- training ------------------------------------------------------------------------------------------------------

GRAD_CASES = [
    ("f40_relu256_tf32", SMALL, [256], "relu", {}, 4, 40),
    ("f128_tanh256_f16_rows2048", dict(SMALL, num_features=128), [256], "tanh", {}, 16, 128),
    ("f123_relu256_100_ffma", dict(PYRAMID, num_features=123), [256, 100], "relu", {}, 4, 40),
    ("f40_tanh250_256_content_rows2048", SMALL, [250, 256], "tanh", dict(attention_type="content"), 16, 128),
]


def _grads(rec, batch):
    pkg = package()
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
    return algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))


def _check_grads(cfg, params, batch, cost, grads, tol=1e-4, atol_frac=1e-6):
    """check_grads' bar: the cost to 1e-4, each gradient to tol of its largest entry plus atol_frac of the model's."""
    want_cost, want = BO.cost_and_grads(cfg, params, *batch)
    gmax = max(np.abs(w).max() for w in want.values())
    assert list(grads) == list(want)
    bad = {}
    for k, w in want.items():
        e = float(np.abs(grads[k].astype(np.float64) - w).max() / max(np.abs(w).max(), 1e-30))
        if e > tol + atol_frac * gmax / max(np.abs(w).max(), 1e-30):
            bad[k] = e
    assert abs(cost - want_cost) <= 1e-4 * abs(want_cost), (cost, want_cost)
    assert not bad, bad
    assert all(np.abs(want[BO.linear_name(i) + ".W"]).max() > 0 for i in range(len(cfg["bottom"]["dims"])))


@pytest.mark.parametrize("case,arch,dims,activation,extra,B,T", GRAD_CASES, ids=[c[0] for c in GRAD_CASES])
def test_gradients_match_oracle(case, arch, dims, activation, extra, B, T):
    """Every parameter's gradient against the float64 oracle: the bottom's on the split-K tensor-core products at
    T * B >= 2048 rows and width a multiple of 128, on FFMA tiles otherwise."""
    _torch()
    cfg = _config(arch, dims, activation, **extra)
    params = _params(cfg, seed=21)
    batch = O.synthetic_batch(cfg, B=B, T=T, seed=22)
    assert not BO.kinks(cfg, params, batch[0], batch[1]), case
    rec = _recognizer(cfg, params)
    cost, grads = _grads(rec, batch)
    _check_grads(cfg, params, batch, cost, grads)


def test_two_optimizer_steps_match_train_step():
    """process_batch twice (momentum + AdaDelta + max-norm, which the bottom's W is subject to, + decay) == two oracle
    train_steps: cost, gradient norm and every parameter after each step."""
    _torch()
    pkg = package()
    cfg = _config(SMALL, [256, 100], "relu")
    params = _params(cfg, seed=31)
    tc = G.make_train_config(gradient_threshold=2.0, scale=0.05, momentum=0.5, decay_rate=0.95, epsilon=1e-6,
                             max_norm=1.0, decay=1e-4)
    rec = _recognizer(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(tc, dict(max_norm=tc["max_norm"])),
                               decay=tc["decay"])
    algo.initialize()
    ref = OrderedDict((k, v.astype(np.float64)) for k, v in params.items())
    state = {}
    for step in range(2):
        batch = O.synthetic_batch(cfg, B=4, T=40, seed=100 + step)
        assert not BO.kinks(cfg, {k: v for k, v in ref.items()}, batch[0], batch[1])
        penalty = tc["decay"] * sum(float((v ** 2).sum()) for k, v in ref.items() if G.is_weight(k))
        ref, ref_cost, ref_grads = BO.train_step(cfg, ref, state, batch, tc)
        algo.process_batch(dict(zip(algo.SOURCES, batch)))
        assert abs(float(algo.last_cost.item()) - (ref_cost - penalty)) <= 1e-4 * abs(ref_cost - penalty), step
        norm = G.l2_norm(ref_grads.values())
        assert abs(algo.total_gradient_norm() - norm) <= 1e-4 * norm, step
        got = rec.get_parameter_values()
        for k, v in ref.items():
            assert np.abs(got[k] - v).max() <= 2e-5 * max(1.0, np.abs(v).max()) + 1e-6, (step, k)
    W = rec.get_parameter_values()[BO.linear_name(0) + ".W"].astype(np.float64)
    assert (np.sqrt((W ** 2).sum(axis=0)) <= 1.0 + 1e-5).all()


def test_one_step_under_adaptive_noise():
    """With adaptive noise the step runs on the noisy parameters, bottom included: its cost and gradients are the
    oracle's at the noisy parameters the library reports, and the bottom has log-variances of its own."""
    torch = _torch()
    pkg = package()
    cfg = _config(SMALL, [256], "tanh")
    params = _params(cfg, seed=41)
    rec = _recognizer(cfg, params)
    tc = G.make_train_config(gradient_threshold=2.0, scale=0.05, momentum=0.5, decay_rate=0.95, epsilon=1e-6,
                             max_norm=1.0)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(tc, dict(max_norm=1.0)),
                               adaptive_noise=dict(num_examples=100, init_sigma=1e-2, model_cost_coefficient=1.0,
                                                   seed=7))
    algo.initialize()
    batch = O.synthetic_batch(cfg, B=4, T=40, seed=42)
    assert "/adaptive_noise." + BO.linear_name(0)[1:] + ".W" in algo.noise_parameter_values()
    algo._forward_backward(dict(zip(algo.SOURCES, batch)), None)
    lib, h = pkg._lib.load(), rec._require_ready()
    noisy = torch.zeros((algo._n,), dtype=torch.float32, device=rec.device)
    pkg._lib.check(lib.lvsr_train_noise_params(h, noisy.data_ptr(), rec._stream()))
    torch.cuda.synchronize()
    flat, raw = noisy.cpu().numpy(), algo._buf[:algo._n].cpu().numpy()
    shapes = rec.parameter_shapes()
    at = OrderedDict((k, flat[o:o + c].reshape(shapes[k]).astype(np.float64)) for k, (o, c) in algo._offsets().items())
    grads = OrderedDict((k, raw[o:o + c].reshape(shapes[k])) for k, (o, c) in algo._offsets().items())
    W = BO.linear_name(0) + ".W"
    assert 0 < np.abs(at[W] - params[W]).max() < 0.1
    _check_grads(cfg, at, batch, float(algo._cost.item()), grads)
    algo.process_batch(dict(zip(algo.SOURCES, batch)))
    assert np.isfinite(float(algo.last_cost.item()))


@pytest.mark.parametrize("activation", ["relu", "tanh"])
def test_padded_frames_do_not_matter(activation):
    """Padded frames holding values around 1e3 give the cost and every gradient bit for bit of the same batch padded
    with zeros: the BiGRU backward gives those frames exactly zero dPre, so the bottom's backward adds nothing."""
    _torch()
    cfg = _config(PYRAMID, [256, 100], activation)
    params = _params(cfg, seed=51)
    x, m, labels, lm = O.synthetic_batch(cfg, B=4, T=40, seed=52)
    assert (m == 0).any()
    zero = np.where(m[:, :, None] > 0, x, 0.0)
    loud = np.where(m[:, :, None] > 0, x, 1e3 * (1 + np.random.RandomState(0).rand(*x.shape)))
    rec = _recognizer(cfg, params)
    c0, g0 = _grads(rec, (zero, m, labels, lm))
    c1, g1 = _grads(rec, (loud, m, labels, lm))
    assert c0 == c1
    for k in g0:
        assert np.array_equal(g0[k], g1[k]), k


def test_checkpoint_round_trip(tmp_path):
    """save_params writes the bottom under its Blocks names; load_params of that checkpoint fills them in a fresh
    recognizer, which then computes the same costs."""
    _torch()
    cfg = _config(SMALL, [256], "relu")
    params = _params(cfg, seed=61)
    rec = _recognizer(cfg, params)
    path = str(tmp_path / "model.tar")
    rec.save_params(path)
    values = rec.load_checkpoint_values(path)
    assert np.array_equal(values[BO.linear_name(0) + ".W"], params[BO.linear_name(0) + ".W"])
    fresh = _recognizer(cfg)
    fresh.initialize()
    report = fresh.load_params(path)
    assert report == dict(unknown=[], missing=[])
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=30, seed=62)
    assert np.array_equal(fresh.cost(x, m, labels, lm), rec.cost(x, m, labels, lm))


def test_compat_train_and_search(tmp_path, capsys):
    """compat's train then search with bottom.dims [64] (Rectifier) from the YAML."""
    _torch()
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as LC
    import lvsr.main as M
    exp = write_experiment(tmp_path)
    cfg = LC.Configuration(exp["base"], "$LVSR/lvsr/configs/schema.yaml", [("net.bottom.dims", "[64]")])
    out = os.path.join(str(tmp_path), "model.tar")
    M.train(cfg, out)
    capsys.readouterr()
    single = LC.Configuration(exp["base"], "$LVSR/lvsr/configs/schema.yaml",
                              [("net.bottom.dims", "[64]"), ("monitoring.search.beam_size", "2")])
    M.search(single, None, out, "valid", None, None, str(tmp_path / "decoded.txt"), False, 1)
    assert "Average CER:" in capsys.readouterr().out
    values = package().SpeechRecognizer.load_checkpoint_values(out)
    assert values[BO.linear_name(0) + ".W"].shape == (40, 64)
