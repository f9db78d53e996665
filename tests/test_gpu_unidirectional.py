"""Unidirectional encoders (net.bidir: False) on the GPU, against the float64 oracle of tests/unidirectional_oracle.py:

* the encoder output at every width 64 .. 512 (one row of one frame, 33 ragged rows, 64 rows over 300 steps) and the
  pyramid [192, 448] subsampled [1, 2]; row counts that leave 4- and 8-row clusters partly empty and need more than
  one wave of them, at T = 1 and with ragged masks; the same under LVSR_NO_TC_GEMM=1.  Each case reads back the plan:
  one cluster per RB rows (no backward clusters), the scan kernel, and the projection path (fp16 wgmma where 3 D is a
  multiple of 128, FFMA at 64, 192, 320 and 448);
* teacher-forced costs at E = 64, 192, 320 and 448 with both attention types, as planned and under LVSR_NO_DEC_SCAN=1:
  the persistent decoder needs kper_ok(E + C) and kper_ok(C), which only multiples of 128 meet, so both run the
  step-wise kernels; greedy steps; search_many token for token against the oracle's BeamSearch;
* gradients at [256] (tensor-core weight gradients), [448] (FFMA), the pyramid and content attention; two optimizer
  steps; dropout and adaptive noise repeat bit for bit; save_params / load_params; the streamed projection of a
  4 x 256 forward-only encoder, whose claims must only take final rows.

The bounds are the ones the bidirectional files use: 1e-4 of the output's range for the encoder output and the costs,
helpers.check_grads' for the gradients."""
import os

import numpy as np
import pytest

import unidirectional_oracle as U
from helpers import O, PYRAMID, check_overlap_claims, elementwise_err, f32, make_recognizer, package, rel_err
from helpers import check_unidirectional_grads as _grads
from oracle import lvsr_oracle_grad as G

pytestmark = pytest.mark.gpu

OUT_TOL = 1e-4
WIDTHS = [64, 128, 192, 256, 320, 384, 448, 512]


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _config(dims, sub=None, attention="content_and_conv", **kw):
    arch = dict(PYRAMID, dims_bidir=dims, subsample=sub or [1] * len(dims))
    arch.update(kw)
    return U.make_config(attention_type=attention, **arch)


def _rec(cfg, params):
    return make_recognizer(cfg, params, bidir=False)


def _check_plan(p, D, B, T, K):
    """One cluster of RB rows each (forward only); the scan kernel of the width; the projection's path."""
    kernel = "mma" if D == 256 and os.environ.get("LVSR_BIGRU_MMA", "1") != "0" else "ffma"
    assert p["bigru"] == kernel and p["T"] == T, p
    assert p["rb"] in ((4, 8) if kernel == "mma" else (4,)), p
    assert p["cs"] == (4 if kernel == "mma" else D // 32), p
    assert p["clusters"] == -(-B // p["rb"]), p
    assert p["resident"] > 0 and p["waves"] == -(-p["clusters"] // p["resident"]), p
    tc = os.environ.get("LVSR_NO_TC_GEMM") is None and (3 * D) % 128 == 0
    assert p["proj"] == ("tc" if tc else "ffma"), p
    if tc:
        assert p["operands"] == ("f16x3" if K % 64 == 0 else "tf32x3"), p


def _encode(cfg, params, x, m):
    rec = _rec(cfg, params)
    att, attm = rec.encode(x, m)
    want, wmask = U.encoder(cfg, params, x, m)
    assert att.shape[2] == cfg["dims_bidir"][-1] == rec.dim_encoded
    assert np.array_equal(attm.cpu().numpy(), wmask.astype(np.float32))
    got = att.cpu().numpy()
    return rec, rel_err(got, want), elementwise_err(got, want)


def _batch(cfg, B, T, seed, one_frame=False):
    x, m, _, _ = O.synthetic_batch(cfg, B=B, T=T, seed=seed, min_frac=0.3)
    if one_frame:
        m[:, 0] = np.arange(T) < 1
        x *= m[:, :, None]
    return f32(x), m


def _check_layers(rec, cfg, B, T):
    Tl, K = T, cfg["num_features"]
    for l, p in enumerate(rec.encoder_plan()):
        _check_plan(p, cfg["dims_bidir"][l], B, Tl, K)
        K, Tl = cfg["dims_bidir"][l], -(-Tl // cfg["subsample"][l])


@pytest.mark.parametrize("D", WIDTHS)
def test_encoder_output_per_width(D):
    _torch()
    cfg = _config([D])
    params = {k: f32(v) for k, v in U.init_params(cfg, seed=D, scale=10.0).items()}
    for B, T, one_frame in ((1, 1, False), (33, 40, True), (64, 300, False)):
        x, m = _batch(cfg, B, T, D + B, one_frame)
        rec, err, eerr = _encode(cfg, params, x, m)
        print("D=%d B=%d T=%d: %.2e (per element %.2e)" % (D, B, T, err, eerr), rec.encoder_plan()[0])
        _check_layers(rec, cfg, B, T)
        assert err < OUT_TOL, (B, T, err)


def test_encoder_output_pyramid():
    _torch()
    cfg = _config([192, 448], [1, 2])
    params = {k: f32(v) for k, v in U.init_params(cfg, seed=7, scale=10.0).items()}
    x, m = _batch(cfg, 33, 61, 61, one_frame=True)
    rec, err, eerr = _encode(cfg, params, x, m)
    print("pyramid %.2e (per element %.2e)" % (err, eerr), rec.encoder_plan())
    _check_layers(rec, cfg, 33, 61)
    assert err < OUT_TOL, err


@pytest.mark.parametrize("no_tc", [False, True], ids=["tc", "no_tc_gemm"])
@pytest.mark.parametrize("D", [64, 256, 448])
def test_encoder_output_partial_clusters_and_waves(D, no_tc, monkeypatch):
    """B = 5, 37 and 131 leave the last 4- or 8-row cluster partly empty; 4 * 133 rows of the 256-unit tensor-core
    scan need more than one wave of clusters; T = 1 and ragged masks."""
    _torch()
    if no_tc:
        monkeypatch.setenv("LVSR_NO_TC_GEMM", "1")
    cfg = _config([D])
    params = {k: f32(v) for k, v in U.init_params(cfg, seed=D + 3, scale=10.0).items()}
    waves = []
    for B, T in ((5, 1), (37, 9), (131, 1), (4 * 133, 3)):
        x, m = _batch(cfg, B, T, B + T, one_frame=(T > 1))
        rec, err, eerr = _encode(cfg, params, x, m)
        p = rec.encoder_plan()[0]
        print("D=%d B=%d T=%d: %.2e" % (D, B, T, err), p)
        _check_layers(rec, cfg, B, T)
        waves.append(p["waves"])
        assert err < OUT_TOL, (B, T, err)
    if D == 256:
        assert max(waves) > 1, waves


# ---- costs, greedy steps and search at the new encoded widths ---------------------------------------------------------

@pytest.mark.parametrize("attention", ["content_and_conv", "content"])
@pytest.mark.parametrize("E", [64, 192, 320, 448])
@pytest.mark.parametrize("stepwise", [False, True], ids=["planned", "no_dec_scan"])
def test_costs_at_new_encoded_widths(E, attention, stepwise, monkeypatch):
    _torch()
    if stepwise:
        monkeypatch.setenv("LVSR_NO_DEC_SCAN", "1")
    cfg = _config([E], attention=attention)
    params = {k: f32(v) for k, v in U.init_params(cfg, seed=E, scale=10.0).items()}
    x, m, labels, lm = O.synthetic_batch(cfg, B=5, T=50, seed=E + 1)
    x = f32(x)
    rec = _rec(cfg, params)
    got = rec.cost(x, m, labels, lm)
    want = U.recognizer_cost(cfg, params, x, m, labels, lm)
    err = rel_err(got, want)
    plan = rec.decoder_plan()
    print("E=%d %s %s: %.2e" % (E, attention, "step-wise" if stepwise else "planned", err), plan)
    # the persistent decoder needs kper_ok(E + C) and kper_ok(C), so E a multiple of 128: at these widths the planner
    # takes the step-wise kernels, as LVSR_NO_DEC_SCAN=1 forces them
    assert plan["kernel"] == "stepwise" and not plan["ran"] and plan["att_cs"] >= 1, plan
    assert rec.launch_status()[0] == 0
    assert err < OUT_TOL, err


@pytest.mark.parametrize("E", [64, 448])
def test_greedy_steps(E):
    torch = _torch()
    cfg = _config([E])
    params = {k: f32(v) for k, v in U.init_params(cfg, seed=E + 2, scale=10.0).items()}
    x, m = _batch(cfg, 3, 40, E)
    rec = _rec(cfg, params)
    att, attm = rec.encode(x, m)
    ctx = dict(attended=att, attended_mask=attm)
    a64, m64 = U.encoder(cfg, params, x, m)
    st_o = U.initial_states(cfg, params, 3, a64)
    st_g = rec._initial_states(att.shape[0], 3)
    for step in range(5):
        lp_o = U.logprobs_computer(cfg, params, a64, m64, st_o)
        lp_g = rec._logprobs(ctx, st_g).double().cpu().numpy()
        err = elementwise_err(lp_g, lp_o)
        print("E=%d step %d logprobs %.2e" % (E, step, err))
        assert err < 1e-4, (step, err)
        y = lp_o.argmin(axis=1)
        st_o = U.next_state_computer(cfg, params, a64, m64, st_o, y)
        st_g = rec._next_states(ctx, st_g, y)
        assert elementwise_err(st_g["states"].double().cpu().numpy(), st_o["states"]) < 1e-4


@pytest.mark.parametrize("attention", ["content_and_conv", "content"])
def test_search_many_matches_oracle(attention):
    _torch()
    scale, beam = 2.0, 5
    cfg = _config([192, 320], attention=attention, max_decoded_length_scale=scale)
    params = U.init_params(cfg, seed=31, scale=10.0)
    # a peaky readout with an end-of-sequence bias, so that every utterance finishes hypotheses
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.W"] *= 4.0
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.b"][cfg["eos_label"]] = 4.0
    params = {k: f32(v) for k, v in params.items()}
    rng = np.random.RandomState(5)
    utts = [f32(rng.normal(size=(T, cfg["num_features"]))) for T in (36, 25, 30)]
    rec = _rec(cfg, params)
    rec.init_beam_search(beam)
    got = rec._beam_search.search_many([u.astype(np.float32) for u in utts], cfg["eos_label"],
                                       [int(u.shape[0] / scale) for u in utts], raise_on_failure=False)
    for u, g in zip(utts, got):
        want = U.beam_search(cfg, params, u, beam)
        assert g is not None and want, (g, want)
        assert list(g[0][0]) == list(want[0][0]), (g[0], want[0])
        assert abs(g[1][0] - float(want[1][0])) <= 1e-4 * max(1.0, abs(float(want[1][0]))), (g[1], want[1])
    assert [p["cs"] for p in rec.encoder_plan()] == [6, 10]


# ---- training ----------------------------------------------------------------------------------------------------------

GRADS = {                 # name -> (widths, subsampling, B, T, attention)
    "d256_tc": ([256], [1], 33, 63, "content_and_conv"),
    "d448_ffma": ([448], [1], 4, 40, "content_and_conv"),
    "pyramid_192_448": ([192, 448], [1, 2], 5, 41, "content_and_conv"),
    "d320_content": ([320], [1], 4, 32, "content"),
}


@pytest.mark.parametrize("case", sorted(GRADS))
def test_gradients(case):
    _torch()
    dims, sub, B, T, attention = GRADS[case]
    cfg = _config(dims, sub, attention=attention)
    params = {k: f32(v) for k, v in U.init_params(cfg, seed=len(case), scale=10.0).items()}
    x, m, labels, lm = O.synthetic_batch(cfg, B=B, T=T, seed=B + T)
    rec = _grads(cfg, params, (f32(x), m, labels, lm))
    plan = rec.encoder_plan()
    print(case, [(p["bwd_cs"], p["wgrad"], p["dx"], p["T"]) for p in plan])
    Tl = T
    for l, p in enumerate(plan):
        assert p["bwd_cs"] == dims[l] // 32 and p["tape"], (l, p)
        assert p["wgrad"] == ("tc" if Tl * B >= 2048 and dims[l] % 128 == 0 else "ffma"), (l, p)
        Tl = -(-Tl // sub[l])
    if case == "d256_tc":
        assert plan[0]["wgrad"] == "tc"


def test_two_optimizer_steps():
    _torch()
    from collections import OrderedDict
    cfg = _config([192, 256], [1, 2])
    params = U.init_params(cfg, seed=11, scale=10.0)
    tc = G.make_train_config(gradient_threshold=2.0, rules=("momentum", "adadelta"), scale=0.05, momentum=0.5,
                             decay_rate=0.95, epsilon=1e-6, max_norm=1.0)
    pkg = package()
    rec = _rec(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(tc, dict(max_norm=tc["max_norm"])),
                               decay=tc["decay"])
    algo.initialize()
    ref, state = OrderedDict((k, v.copy()) for k, v in params.items()), {}
    for step in range(2):
        batch = O.synthetic_batch(cfg, B=4, T=40, seed=100 + step)
        ref, ref_cost, ref_grads = U.train_step(cfg, ref, state, batch, tc)
        algo.process_batch(dict(zip(algo.SOURCES, batch)))
        assert abs(float(algo.last_cost.item()) - ref_cost) <= 1e-4 * abs(ref_cost), (step, algo.last_cost.item())
        norm = G.l2_norm(ref_grads.values())
        assert abs(algo.total_gradient_norm() - norm) <= 1e-4 * norm
        got = rec.get_parameter_values()
        for k, v in ref.items():
            assert np.abs(got[k] - v).max() <= 2e-5 * max(1.0, np.abs(v).max()) + 1e-6, (step, k)


@pytest.mark.parametrize("kind", ["dropout", "adaptive_noise"])
def test_regularised_steps_repeat_bit_for_bit(kind):
    _torch()
    cfg = _config([192, 256], [1, 2])
    params = U.init_params(cfg, seed=13, scale=10.0)
    tc = G.make_train_config(gradient_threshold=2.0, rules=("momentum",), scale=0.05, momentum=0.5, max_norm=1.0)
    pkg = package()
    batch = O.synthetic_batch(cfg, B=4, T=40, seed=3)

    def run():
        rec = _rec(cfg, params)
        extra = (dict(regularization=dict(dropout=True, seed=5)) if kind == "dropout" else
                 dict(adaptive_noise=dict(num_examples=40, init_sigma=1e-2, model_cost_coefficient=0.5, seed=7)))
        algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(tc, dict(max_norm=1.0)),
                                   **extra)
        algo.initialize()
        algo.process_batch(dict(zip(algo.SOURCES, batch)))
        return float(algo.last_cost.item()), rec.get_parameter_values()

    c1, p1 = run()
    c2, p2 = run()
    assert np.isfinite(c1) and c1 == c2
    for k in p1:
        assert np.array_equal(p1[k], p2[k]), k
    assert any(not np.array_equal(p1[k], np.asarray(params[k], np.float32)) for k in p1)


def test_save_and_load_params(tmp_path):
    _torch()
    cfg = _config([192])
    params = U.init_params(cfg, seed=17, scale=10.0)
    rec = _rec(cfg, params)
    path = str(tmp_path / "uni.tar")
    rec.save_params(path)
    names = sorted(rec.load_checkpoint_values(path))
    assert names == sorted(U.param_shapes(cfg)) and any("/with_fork0/" in n for n in names)
    other = _rec(cfg, U.init_params(cfg, seed=18))
    assert other.load_params(path) == dict(unknown=[], missing=[])
    got = other.get_parameter_values()
    for k, v in params.items():
        assert np.array_equal(got[k], np.asarray(v, np.float32)), k


def test_streamed_projection_of_a_forward_only_wsj_encoder():
    """4 x 256 forward-only layers at B = 64: layers 1 .. 3 stream their projection beside the tensor-core scan; the
    output is bit-identical with the streaming off and every claimed tile had final rows."""
    _torch()
    cfg = _config([256, 256, 256, 256], [1, 1, 2, 2], dim_dec=256, dim_matcher=512)
    params = {k: f32(v) for k, v in U.init_params(cfg, seed=19, scale=10.0).items()}
    x, m = _batch(cfg, 64, 200, 1)
    rec = _rec(cfg, params)
    att, _ = rec.encode(x, m)
    plan = rec.encoder_plan()
    print([(p["overlap"], p["tiles_beside"], p["tiles_after"], p["clusters"], p["waves"]) for p in plan])
    assert plan[0]["clusters"] == 16 and plan[0]["waves"] == 1, plan[0]
    check_overlap_claims(rec, plan, 64, cfg["subsample"], ndir=1)
    os.environ["LVSR_ENC_OVERLAP"] = "0"
    try:
        att0, _ = _rec(cfg, params).encode(x, m)
    finally:
        del os.environ["LVSR_ENC_OVERLAP"]
    assert np.array_equal(att.cpu().numpy(), att0.cpu().numpy())
    want, _ = U.encoder(cfg, params, x, m)
    assert rel_err(att.cpu().numpy(), want) < OUT_TOL


def test_compat_train_and_search(tmp_path, capsys):
    """compat's train then search with net.bidir False from the YAML: the checkpoint holds with_fork parameters."""
    import sys
    from compat_helpers import COMPAT, write_experiment
    _torch()
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as LC
    import lvsr.main as M
    exp = write_experiment(tmp_path)
    changes = [("net.bidir", "False"), ("net.dims_bidir", "[192]")]
    cfg = LC.Configuration(exp["base"], "$LVSR/lvsr/configs/schema.yaml", changes)
    out = os.path.join(str(tmp_path), "model.tar")
    M.train(cfg, out)
    capsys.readouterr()
    single = LC.Configuration(exp["base"], "$LVSR/lvsr/configs/schema.yaml",
                              changes + [("monitoring.search.beam_size", "2")])
    M.search(single, None, out, "valid", None, None, str(tmp_path / "decoded.txt"), False, 1)
    assert "Average CER:" in capsys.readouterr().out
    values = package().SpeechRecognizer.load_checkpoint_values(out)
    assert values["/recognizer/encoder/with_fork0/fork/fork_inputs.W"].shape == (40, 192)
    assert not any("/bidir0/" in k for k in values)
