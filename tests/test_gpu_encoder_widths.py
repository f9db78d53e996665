"""Encoder widths beyond 128 / 256 on the GPU: every dims_bidir entry that is a multiple of 64 from 64 to 512 runs the
FFMA BiGRU scan with 32 units per CTA (clusters of D / 32 CTAs, non-portable above 8) and its reverse-time twin, against
the float64 oracle (oracle/lvsr_oracle.py, oracle/lvsr_oracle_grad.py):

* the encoder output, per width 64, 192, 320, 384, 448 and 512, on one row of one frame, 33 rows holding a one-frame
  utterance and the metric batch of 64 rows over 300 steps; two pyramids ([192, 320, 512] subsampled [1, 2, 2] and
  [512, 64]); the kernel, rows and CTAs per cluster, clusters, resident clusters and waves read back from encoder_plan();
* every parameter's gradient (helpers.check_grads, the bar of test_gpu_train_configs.py) at 64, 320, 512 -- T*B >= 2048
  there, so its weight gradients run on tensor cores, while 320 takes the FFMA tiles -- and a mixed pyramid; two optimizer
  steps at 384; one adaptive-noise step at 320;
* beam search at 320 with content and content_and_conv attention, token for token;
* the persistent decoder at E = 640 (dim_dec 128: kper_ok(E + C) holds);
* the encoder overlap, with a 192- and a 320-unit layer behind a tensor-core 256-unit one: bit-identical either way;
* refusals before any work: widths 250, 96 and 576, and a training step at E = 1024 one frame longer than the
  attention backward's shared memory holds.

Worst errors measured on an H100 80GB HBM3 (700 W power limit): encoder output of one layer 9.9e-7 of its range (8.1e-6
per element, D = 512, B = 64, T = 300), pyramids 8.0e-6 ([512, 64]; 6.8e-5 per element); gradients 4.8e-5 of a
parameter's largest entry (the [192, 320, 512] pyramid), 4.9e-6 at a single layer; the E = 640 cost 1.4e-7, on the
persistent decoder.  The bound is 1e-4 throughout (check_grads' own for the gradients)."""
import numpy as np
import pytest

import content_oracle as CO
from helpers import O, PYRAMID, WSJ, check_grads, elementwise_err, f32, make_recognizer, package, rel_err, \
    train_like_the_oracle
from oracle import lvsr_oracle_grad as G

pytestmark = pytest.mark.gpu

OUT_TOL = 1e-4           # encoder output: max |error| over its largest magnitude
WIDTHS = [64, 192, 320, 384, 448, 512]


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _encode_case(cfg, params, B, T, seed, one_frame):
    params = {k: f32(v) for k, v in params.items()}
    x, m, _, _ = O.synthetic_batch(cfg, B=B, T=T, seed=seed, min_frac=0.3)
    if one_frame:
        m[:, 0] = np.arange(T) < 1
        x *= m[:, :, None]
    x = f32(x)
    rec = make_recognizer(cfg, params)
    att, attm = rec.encode(x, m)
    want, wmask = O.encoder(cfg, params, x, m)
    assert np.array_equal(attm.cpu().numpy(), wmask.astype(np.float32))
    got = att.cpu().numpy()
    return rec, rel_err(got, want), elementwise_err(got, want)


def _check_scan_plan(p, D, B, T):
    clusters = 2 * -(-B // 4)
    assert (p["bigru"], p["rb"], p["cs"], p["T"], p["clusters"]) == ("ffma", 4, D // 32, T, clusters), p
    assert p["resident"] > 0 and p["waves"] == -(-clusters // p["resident"]), p


@pytest.mark.parametrize("D", WIDTHS)
def test_encoder_output_per_width(D):
    _torch()
    cfg = O.make_config(**dict(PYRAMID, dims_bidir=[D], subsample=[1]))
    params = O.init_params(cfg, seed=D, scale=10.0)
    for B, T, one_frame in ((1, 1, False), (33, 40, True), (64, 300, False)):
        rec, err, eerr = _encode_case(cfg, params, B, T, seed=D + B, one_frame=one_frame)
        p = rec.encoder_plan()[0]
        print("D=%d B=%d T=%d: %.2e (per element %.2e)" % (D, B, T, err, eerr), p)
        _check_scan_plan(p, D, B, T)
        assert err < OUT_TOL, (B, T, err)


@pytest.mark.parametrize("dims,sub", [([192, 320, 512], [1, 2, 2]), ([512, 64], [1, 1])], ids=["192_320_512", "512_64"])
def test_encoder_output_pyramids(dims, sub):
    _torch()
    cfg = O.make_config(**dict(PYRAMID, dims_bidir=dims, subsample=sub))
    params = O.init_params(cfg, seed=len(dims), scale=10.0)
    T, B = 61, 33
    rec, err, eerr = _encode_case(cfg, params, B, T, seed=T, one_frame=True)
    plan = rec.encoder_plan()
    print(dims, "%.2e (per element %.2e)" % (err, eerr), [(p["T"], p["cs"], p["resident"], p["waves"]) for p in plan])
    Tl = T
    for l, p in enumerate(plan):
        _check_scan_plan(p, dims[l], B, Tl)
        Tl = -(-Tl // sub[l])
    assert err < OUT_TOL, err


# ---- the training step ------------------------------------------------------------------------------------------------

GRADS = {                         # name -> (widths, subsampling, B, T)
    "d64": ([64], [1], 4, 40),
    "d320": ([320], [1], 4, 40),
    "d512_tc": ([512], [1], 8, 256),
    "pyramid_192_320_512": ([192, 320, 512], [1, 2, 2], 5, 61),
}


@pytest.mark.parametrize("case", sorted(GRADS))
def test_gradients(case):
    _torch()
    dims, sub, B, T = GRADS[case]
    cfg = O.make_config(**dict(PYRAMID, dims_bidir=dims, subsample=sub))
    params = {k: f32(v) for k, v in O.init_params(cfg, seed=len(case), scale=10.0).items()}
    x, m, labels, lm = O.synthetic_batch(cfg, B=B, T=T, seed=B + T)
    _, rec = check_grads(cfg, params, (f32(x), m, labels, lm))
    plan = rec.encoder_plan()
    print(case, [(p["bwd_cs"], p["wgrad"], p["T"]) for p in plan])
    Tl = T
    for l, p in enumerate(plan):
        assert p["bwd_cs"] == dims[l] // 32 and p["tape"], (l, p)
        tc = Tl * B >= 2048 and dims[l] % 128 == 0
        assert p["wgrad"] == ("tc" if tc else "ffma"), (l, p)
        Tl = -(-Tl // sub[l])
    if case == "d512_tc":
        assert plan[0]["wgrad"] == "tc"


def test_two_optimizer_steps_at_384():
    _torch()
    cfg = O.make_config(**dict(PYRAMID, dims_bidir=[384], subsample=[1]))
    params = O.init_params(cfg, seed=384, scale=10.0)
    tc = G.make_train_config(gradient_threshold=2.0, rules=("momentum", "adadelta"), scale=0.05, momentum=0.5,
                             decay_rate=0.95, epsilon=1e-6, max_norm=1.0)
    rec, _, _ = train_like_the_oracle(cfg, params, tc, B=4, T=32)
    assert rec.encoder_plan()[0]["bwd_cs"] == 12


def test_adaptive_noise_step_at_320():
    """One process_batch with adaptive weight noise == the oracle's update on the replayed eps (the bar of
    test_gpu_adaptive_noise.py)."""
    torch = _torch()
    import adaptive_noise_oracle as AN
    n_examples, coef = 40, 0.5
    cfg = O.make_config(**dict(PYRAMID, dims_bidir=[320], subsample=[1]))
    params = O.init_params(cfg, seed=5, scale=10.0)
    tc = G.make_train_config(gradient_threshold=2.0, rules=("momentum", "adadelta"), scale=0.05, momentum=0.5,
                             decay_rate=0.95, epsilon=1e-6, max_norm=1.0)
    pkg = package()
    rec = make_recognizer(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(tc, dict(max_norm=tc["max_norm"])),
                               adaptive_noise=dict(num_examples=n_examples, init_sigma=1e-2,
                                                   model_cost_coefficient=coef, seed=7))
    algo.initialize()
    lib, h = pkg._lib.load(), rec._require_ready()
    buf = torch.full((algo._n,), 7.0, dtype=torch.float32, device=rec.device)
    pkg._lib.check(lib.lvsr_train_noise_sample(h, 0, buf.data_ptr(), rec._stream()))
    flat = buf.cpu().numpy()
    shapes = rec.parameter_shapes()
    eps = {k: flat[o:o + c].reshape(shapes[k]).astype(np.float64) for k, (o, c) in algo._offsets().items()}
    ref = {k: np.asarray(v, np.float32).astype(np.float64) for k, v in params.items()}
    batch = O.synthetic_batch(cfg, B=3, T=32, seed=100)
    ref, ls2, cost, _, norm = AN.train_step(cfg, ref, AN.init_ls2(ref, 1e-2), {}, batch, tc, eps, n_examples, coef)
    algo.process_batch(dict(zip(algo.SOURCES, batch)))
    assert abs(float(algo.last_cost.item()) - cost) <= 1e-4 * abs(cost), (algo.last_cost.item(), cost)
    assert abs(algo.total_gradient_norm() - norm) <= 1e-4 * norm, (algo.total_gradient_norm(), norm)
    got, got_ls2 = rec.get_parameter_values(), algo.noise_parameter_values()
    for k, v in ref.items():
        assert np.abs(got[k] - v).max() <= 1e-4 * np.abs(v).max(), k
        assert np.abs(got_ls2[AN.noise_name(k)] - ls2[k]).max() <= 1e-4 * np.abs(ls2[k]).max(), k


# ---- search and the persistent decoder ----------------------------------------------------------------------------------

@pytest.mark.parametrize("attention", ["content_and_conv", "content"])
def test_beam_search_at_320(attention):
    _torch()
    M = CO if attention == "content" else O
    cfg = M.make_config(**dict(PYRAMID, dims_bidir=[320, 320, 320], max_decoded_length_scale=3.0))
    # a peaky readout with a strong end-of-sequence bias: the oracle finishes two of the three utterances, with 2 to 7
    # hypotheses each
    params = M.init_params(cfg, seed=12, scale=10.0)
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.W"] *= 5.0
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.b"][cfg["eos_label"]] = 6.0
    rng = np.random.RandomState(5)
    utts = [rng.normal(size=(T, cfg["num_features"])) for T in (64, 37, 52)]
    rec = make_recognizer(cfg, params)
    rec.init_beam_search(5)
    got = rec._beam_search.search_many([u.astype(np.float32) for u in utts], cfg["eos_label"],
                                       [int(u.shape[0] / 3.0) for u in utts], raise_on_failure=False)
    n_found = 0
    for u, g in zip(utts, got):
        try:
            want = M.beam_search(cfg, params, u, 5)
        except O.CandidateNotFoundError:
            assert g is None
            continue
        assert g is not None and g[0] == want[0]
        n_found += 1
    assert n_found >= 2
    assert rec.encoder_plan()[0]["cs"] == 10


def test_persistent_decoder_at_e640():
    _torch()
    cfg = O.make_config(**dict(PYRAMID, dims_bidir=[320], subsample=[1], dim_dec=128, dim_matcher=256))
    params = {k: f32(v) for k, v in O.init_params(cfg, seed=3, scale=10.0).items()}
    x, m, labels, lm = O.synthetic_batch(cfg, B=8, T=48, seed=4)
    rec = make_recognizer(cfg, params)
    got = rec.cost(f32(x), m, labels, lm)
    want = O.recognizer_cost(cfg, params, f32(x), m, labels, lm)
    plan = rec.decoder_plan()
    print("E=640 cost %.2e" % rel_err(got, want), plan)
    # kper_ok(640 + 128) and kper_ok(128) hold: the persistent decoder, unless its planner finds no cluster shape
    assert plan["kernel"].startswith("dec_scan") if plan["ran"] else plan["kernel"] == "stepwise", plan
    assert rel_err(got, want) < 1e-4


# ---- the encoder overlap ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("D1", [192, 320])
def test_encoder_overlap_behind_a_tensor_core_layer(D1, monkeypatch):
    from test_gpu_encoder_overlap import _case
    plan = _case(dict(dims_bidir=[256, D1], subsample=[1, 1]), 16, 100, D1, monkeypatch, warm=True)
    assert plan[0]["bigru"] == "mma" and plan[1]["overlap"] and plan[1]["cs"] == D1 // 32, plan


# ---- refusals ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("D", [250, 96, 576])
def test_widths_off_the_rule_are_refused(D):
    _torch()
    cfg = O.make_config(**dict(PYRAMID, dims_bidir=[128, D], subsample=[1, 1]))
    with pytest.raises(RuntimeError, match="encoder dim %d of layer 1 unsupported \\(a multiple of 64 from 64 to 512\\)" % D):
        make_recognizer(cfg, O.init_params(cfg, seed=1, scale=10.0))


def test_training_beyond_the_attention_backward_at_e1024_is_refused():
    """At E = 1024 the attention backward's shared memory holds one encoded length less than the longest utterance:
    refused before any work, and the recognizer still trains on a shorter batch afterwards."""
    _torch()
    from test_gpu_train_lengths import _longest_trainable
    cfg = O.make_config(**dict(WSJ, dims_bidir=[512], subsample=[1]))
    tmax = _longest_trainable(cfg["dim_matcher"], 1024, cfg["conv_num_filters"], cfg["conv_n"])
    pkg = package()
    rec = make_recognizer(cfg, O.init_params(cfg, seed=2, scale=10.0))
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
    batch = O.synthetic_batch(cfg, B=2, T=tmax + 1, seed=3)
    batch[1][:, 0] = 1.0                                  # the longest utterance spans all T' = tmax + 1 frames
    with pytest.raises(RuntimeError, match="attention backward: shape unsupported"):
        algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
    cost, _ = algo.cost_and_gradients(dict(zip(algo.SOURCES, O.synthetic_batch(cfg, B=2, T=32, seed=4))))
    assert np.isfinite(cost)
