"""Training step on the GPU against the gradient / optimizer oracle (oracle/lvsr_oracle_grad.py):
gradients of every parameter (1e-4 of the parameter's largest gradient entry + a small absolute floor),
the cost, and parameters after updates with the step-rule chain of lvsr/main.py:480-519."""
import numpy as np
import pytest

from helpers import O, PYRAMID, WSJ, make_recognizer, package, train_like_the_oracle
from helpers import check_grads as _check_grads
from oracle import lvsr_oracle_grad as G

pytestmark = pytest.mark.gpu

FILTERS = "/recognizer/generator/att_trans/conv_att/conv1d.filters"


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


PRIORS = [None, dict(type="window_around_median", before=5, after=7),
          dict(type="expanding", initial_begin=0, initial_end=6, min_speed=0.7, max_speed=2.2)]


@pytest.mark.parametrize("prior", PRIORS, ids=lambda p: "default" if p is None else p["type"])
def test_gradients_match_oracle_pyramid(prior):
    _torch()
    cfg = O.make_config(prior=prior, **PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    batch = O.synthetic_batch(cfg, B=6, T=56, seed=21)
    _check_grads(cfg, params, batch)


def test_gradients_match_oracle_wsj_architecture():
    """4-layer pyramidal BiGRU(256) (8-CTA clusters in the BPTT kernel), M=512, n=100, 2 label-masked rows."""
    _torch()
    cfg = O.make_config(**WSJ)
    params = O.init_params(cfg, seed=1, scale=10.0)
    batch = O.synthetic_batch(cfg, B=5, T=48, seed=3)
    _check_grads(cfg, params, batch)


def test_gradients_island_batch_no_masks():
    """Two 16-row islands of the persistent decoder (cs 1: T' = 10 is too short for larger clusters)."""
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=7, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=32, T=40, seed=12)
    _, rec = _check_grads(cfg, params, (x, None, labels, None))
    plan = rec.decoder_plan()
    assert plan["ran"] and plan["nisl"] == 2 and plan["cs"] == 1, plan


def _params_with_long_filter_columns(cfg, max_norm):
    """Trained-like parameters whose conv filters have columns (axis 0) both longer and shorter than max_norm."""
    params = O.init_params(cfg, seed=5, scale=10.0)
    f = params[FILTERS].copy()
    f[:, ::2] *= 3.0 * max_norm / np.sqrt((f[:, ::2] ** 2).sum(axis=0)).min()
    params[FILTERS] = f
    cols = np.sqrt((f ** 2).sum(axis=0))
    assert (cols[::2] > 2.9 * max_norm).all() and (cols[1::2] < max_norm).all()
    return params


@pytest.mark.parametrize("rules,max_norm", [(("momentum", "adadelta"), 1.0), (("momentum",), 0.0), (("adadelta",), 0.5)])
def test_training_steps_match_oracle(rules, max_norm):
    """Two process_batch calls == two oracle train_steps (float64) on the same batches."""
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    tc = G.make_train_config(gradient_threshold=2.0, rules=rules, scale=0.05, momentum=0.5, decay_rate=0.95,
                             epsilon=1e-6, max_norm=max_norm)
    rec, ref, _ = train_like_the_oracle(cfg, params, tc)
    # the forward pass uses the updated (re-packed) weights
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=32, seed=5)
    want = O.recognizer_cost(cfg, ref, x, m, labels, lm)
    got = rec.cost(x, m, labels, lm)
    assert np.abs(got - want).max() <= 1e-3 * np.abs(want).max()


def test_max_norm_clips_weights_but_not_the_conv_filters():
    """Restrict(VariableClipping(max_norm, axis=0), WEIGHT) (lvsr/main.py:490-505): the conv filters have no WEIGHT role
    (lvsr/bricks/attention.py:31-33), so filter columns far longer than max_norm move exactly as the oracle's, unclipped."""
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = _params_with_long_filter_columns(cfg, 1.0)
    tc = G.make_train_config(gradient_threshold=2.0, rules=("momentum", "adadelta"), scale=0.05, momentum=0.5,
                             decay_rate=0.95, epsilon=1e-6, max_norm=1.0)
    rec, ref, _ = train_like_the_oracle(cfg, params, tc)
    got = rec.get_parameter_values()[FILTERS].astype(np.float64)
    assert (np.sqrt((got[:, ::2] ** 2).sum(axis=0)) > 2.5).all()           # still far above max_norm


def test_weight_decay_with_momentum_adadelta_and_max_norm():
    """decay > 0 (lvsr/main.py:418-420) on the full WSJ chain: 2 decay W joins the gradient of every WEIGHT parameter
    before the clipping norm; biases, initial states and the conv filters are not decayed."""
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = _params_with_long_filter_columns(cfg, 1.0)
    tc = G.make_train_config(gradient_threshold=2.0, rules=("momentum", "adadelta"), scale=0.05, momentum=0.5,
                             decay_rate=0.95, epsilon=1e-6, max_norm=1.0, decay=0.01)
    train_like_the_oracle(cfg, params, tc)


@pytest.mark.parametrize("threshold,active", [(1e-3, True), (1e6, False)], ids=["always_clipped", "never_clipped"])
def test_step_clipping_active_and_inactive(threshold, active):
    """StepClipping (B/algorithms/__init__.py:634-643) with a threshold far below the gradient norm (every step is
    rescaled to norm = threshold) and far above it (the step is the plain gradient)."""
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    tc = G.make_train_config(gradient_threshold=threshold, rules=("momentum",), scale=0.05, momentum=0.5, max_norm=0.0)
    _, _, norms = train_like_the_oracle(cfg, params, tc)
    assert all((n > 100 * threshold) if active else (n < threshold / 100) for n in norms), norms


def test_non_finite_gradient_zeroes_the_parameter_and_burn_in_delays_updates():
    torch = _torch()
    pkg = package()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    batch = O.synthetic_batch(cfg, B=3, T=32, seed=1)
    rec = make_recognizer(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule(
        [pkg.StepClipping(10.0), pkg.Momentum(0.1, 0.0), pkg.RemoveNotFinite(0.0), pkg.BurnIn(num_steps=2)]))
    algo.initialize()
    before = rec.get_parameter_values()
    for i in range(3):
        algo.process_batch(dict(zip(algo.SOURCES, batch)))
        after = rec.get_parameter_values()
        changed = any(np.abs(after[k] - before[k]).max() > 0 for k in before)
        assert changed == (i == 2), i              # lvsr/algorithms.py:35-43: the first num_steps updates are zeroed
    # poison one gradient: RemoveNotFinite(0.0) zeroes that parameter, the others still move (B/algorithms/__init__.py:855-861)
    x = batch[0].copy()
    algo2 = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.Momentum(0.1, 0.0), pkg.RemoveNotFinite(0.0)]))
    algo2.initialize()
    algo2._forward_backward(dict(zip(algo2.SOURCES, (x,) + tuple(batch[1:]))), None)
    name = "/recognizer/generator/readout/post_merge/bias.b"
    import ctypes as C
    lib, h = pkg._lib.load(), rec._require_ready()
    idx = list(rec.parameter_shapes()).index(name)
    off, cnt = C.c_int64(), C.c_int64()
    pkg._lib.check(lib.lvsr_model_param_offset(h, idx, C.byref(off), C.byref(cnt)))
    algo2._buf[off.value] = float("nan")
    pkg._lib.check(lib.lvsr_train_apply_updates(h, algo2._buf.data_ptr(), 1.0, C.byref(algo2._tc), rec._stream()))
    torch.cuda.synchronize()
    now = rec.get_parameter_values()
    assert np.all(now[name] == 0)
    other = "/recognizer/generator/readout/post_merge/mlp/linear_0.W"
    assert np.abs(now[other] - after[other]).max() > 0 and np.isfinite(now[other]).all()


def test_two_gpu_step_equals_single_gpu_step_on_the_concatenated_batch():
    """SURVEY.md 8e: batch sharded over ranks + ONE NCCL all-reduce of the flat gradient buffer."""
    torch = _torch()
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29600 + os.getpid() % 300
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port),
                        os.path.join(root, "tests", "dist_train_worker.py")], capture_output=True, text=True, timeout=600)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "DIST_TRAIN_OK" in r.stdout


def test_gradients_with_tensor_core_backward_gemms(monkeypatch):
    """T*B >= 2048 rows switches the encoder's weight-gradient (X^T dY, split-K) and input-gradient (dY W^T) GEMMs to
    the wgmma 3xTF32 kernel; same bar as the FFMA path, and the two paths agree with each other."""
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    batch = O.synthetic_batch(cfg, B=32, T=64, seed=77)
    algo, rec = _check_grads(cfg, params, batch)
    _, g_tc = algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
    # 2048 rows at layers 0 and 1, 1024 at layer 2
    assert [(p["wgrad"], p["dx"]) for p in rec.encoder_plan()] == [("tc", None), ("tc", "tc"), ("ffma", "tc")]
    monkeypatch.setenv("LVSR_NO_TC_GEMM", "1")
    pkg = package()
    rec2 = make_recognizer(cfg, params)
    algo2 = pkg.GradientDescent(recognizer=rec2, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
    _, g_ff = algo2.cost_and_gradients(dict(zip(algo2.SOURCES, batch)))
    assert [(p["wgrad"], p["dx"]) for p in rec2.encoder_plan()] == [("ffma", None), ("ffma", "ffma"), ("ffma", "ffma")]
    for k in g_tc:
        scale = max(np.abs(g_ff[k]).max(), 1e-30)
        assert np.abs(g_tc[k] - g_ff[k]).max() / scale < 2e-4, k


def test_one_of_n_feedback_cost_and_gradients():
    """embed_outputs=False (the WSJ configs): no lookup table, fork weights indexed by the label."""
    _torch()
    cfg = O.make_config(embed_outputs=False, **PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    assert "/recognizer/generator/fork/fork_inputs.W" in params and params["/recognizer/generator/fork/fork_inputs.W"].shape == (33, 128)
    batch = O.synthetic_batch(cfg, B=5, T=48, seed=9)
    algo, rec = _check_grads(cfg, params, batch)
    want = O.recognizer_cost(cfg, params, *batch)
    got = rec.cost(*batch)
    assert np.abs(got - want).max() <= 1e-4 * np.abs(want).max()


def test_wsj_training_batch_matches_golden_gradients():
    """WSJ architecture, B = 16 (island-mode persistent decoder), T*B = 5120 rows (tensor-core backward GEMMs), against the
    committed float64 gradient oracle (tests/golden/make_train_golden.py): per parameter sum, sum |.|, max |.| and a random
    projection of the gradient."""
    _torch()
    import os
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_golden.npz"))
    cfg = O.make_config(**WSJ)
    params = O.init_params(cfg, seed=1, scale=10.0)
    batch = O.synthetic_batch(cfg, B=16, T=320, seed=17)
    pkg = package()
    rec = make_recognizer(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
    cost, grads = algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
    assert abs(cost - float(gold["cost"])) <= 1e-4 * abs(float(gold["cost"]))
    names, stats = [str(n) for n in gold["names"]], gold["stats"]
    assert names == list(grads)
    rng = np.random.RandomState(7)
    gmax = stats[:, 2].max()
    worst = 0.0
    for k, want in zip(names, stats):
        g = grads[k].astype(np.float64)
        r = rng.normal(size=g.shape)
        got = np.array([g.sum(), np.abs(g).sum(), np.abs(g).max(), (g * r).sum()])
        # sums of n entries of size <= max|g| carry rounding of order sqrt(n) * eps * max|g|; 1e-4 of the natural scale of each statistic
        scale = np.array([want[1], want[1], want[2], want[2] * np.sqrt(g.size)]) + 1e-6 * gmax
        err = np.abs(got - want) / scale
        worst = max(worst, err.max())
        assert (err < 2e-4).all(), (k, err)
    print("worst relative error over %d parameters: %.2e" % (len(names), worst))


def test_single_utterance_single_label_and_determinism():
    """Edge shapes (B = 1, L = 2) and run-to-run determinism: every reduction of the backward pass has a fixed order
    (split-K partials, per-CTA partial sums, no floating-point atomics), so two calls give bit-identical gradients."""
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=1, T=24, seed=2, label_div=24)
    assert labels.shape[0] == 2
    algo, rec = _check_grads(cfg, params, (x, m, labels, lm))
    batch = O.synthetic_batch(cfg, B=32, T=64, seed=3)            # tensor-core split-K path
    pkg = package()
    rec2 = make_recognizer(cfg, params)
    algo2 = pkg.GradientDescent(recognizer=rec2, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
    c1, g1 = algo2.cost_and_gradients(dict(zip(algo2.SOURCES, batch)))
    c2, g2 = algo2.cost_and_gradients(dict(zip(algo2.SOURCES, batch)))
    assert c1 == c2
    for k in g1:
        assert np.array_equal(g1[k], g2[k]), k
