"""The training step bench.py --mode train times (64 utterances of up to 1500 frames on the WSJ architecture, its
first shard's batch and bench.init_values weights) with dropout and with weight noise on:

  * the plans of test_gpu_bench_train.py: the tensor-core BiGRU scan with its tape, tensor-core weight gradients with
    split K, the persistent decoder in B/16 islands, and launch status 0;
  * determinism: a second call at the same update gives bit-identical gradients;
  * dropout keyed by global utterance index inside the step: the batch run as two 32-row shards at utterance offsets
    0 and 32 (lvsr_train_set_utterance_offset) gives the whole batch's gradient, and at offset 0 for both it does not;
  * weight noise re-packed from the means: after a noisy update, the cost of the updated handle equals, bit for bit,
    that of a fresh handle loaded with its parameters, so the tensor-core scan's and the GEMMs' packed operands were
    rebuilt from the means and not from the noisy copy.

The gradients themselves are compared with float64 at these shapes in test_gpu_bench_train.py (no regulariser) and
test_gpu_regularization_paths.py (each regulariser, on the same kernels)."""
import numpy as np
import pytest

import bench
from helpers import bench_recognizer, package

pytestmark = pytest.mark.gpu

TOL, ATOL_FRAC = 1e-4, 1e-6


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _setup(reg):
    pkg = package()
    W = bench.TRAIN_WORKLOAD
    batch = bench.synthetic_batch(**W, seed=bench.shard_seed(0, base=4321))
    rec = bench_recognizer()
    rec.set_parameter_values(bench.init_values(rec.parameter_shapes()))
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(bench.TRAIN_CONF, dict(max_norm=1.0)),
                               regularization=dict(reg, seed=11))
    algo.initialize()
    return algo, rec, batch


def _check_plans(rec, B):
    dec, enc = rec.decoder_plan(), rec.encoder_plan()
    assert rec.launch_status() == (0, 0)
    assert dec["ran"] and dec["kernel"].startswith("dec_scan") and dec["nisl"] == B // 16, dec
    assert all(p["bigru"] == "mma" and p["tape"] for p in enc), enc
    assert all(p["wgrad"] == "tc" and p["wgrad_splits"] > 1 for p in enc), enc


def _sum_of_gradients(algo, batch, offset):
    """The gradient sum of `batch` run as a shard whose first utterance has global index `offset`, flat."""
    algo._forward_backward(dict(zip(algo.SOURCES, batch)), 1.0, offset)
    return algo._buf[:algo._n].double().cpu().numpy()


def _worst(got, want, offsets):
    """Worst error / bar over the parameters: 1e-4 of the parameter's largest |g| plus 1e-6 of the model's."""
    gmax = np.abs(want).max()
    worst = 0.0
    for o, c in offsets.values():
        w, g = want[o:o + c], got[o:o + c]
        worst = max(worst, float(np.abs(g - w).max() / (TOL * np.abs(w).max() + ATOL_FRAC * gmax)))
    return worst


def test_dropout_on_the_benchmarked_step_and_its_shards():
    _torch()
    algo, rec, batch = _setup(dict(dropout=True))
    B = batch[0].shape[1]
    sources = dict(zip(algo.SOURCES, batch))
    cost, grads = algo.cost_and_gradients(sources)
    _check_plans(rec, B)
    cost2, again = algo.cost_and_gradients(sources)
    assert cost2 == cost and all(np.array_equal(again[k], g) for k, g in grads.items())
    full = _sum_of_gradients(algo, batch, 0) / B
    offsets = algo._offsets()
    half = B // 2
    shard = lambda lo: tuple(a[:, lo:lo + half] for a in batch)
    two = (_sum_of_gradients(algo, shard(0), 0) + _sum_of_gradients(algo, shard(half), half)) / B
    worst = _worst(two, full, offsets)
    print("two shards against the whole batch: worst gradient error / bar %.3f" % worst)
    assert worst <= 1.0
    # the second shard keyed as if it were the first draws another mask: the offset reaches the step
    wrong = (_sum_of_gradients(algo, shard(0), 0) + _sum_of_gradients(algo, shard(half), 0)) / B
    assert _worst(wrong, full, offsets) > 10.0


def test_weight_noise_on_the_benchmarked_step_and_the_means_after_an_update():
    _torch()
    algo, rec, batch = _setup(dict(noise=0.05))
    B = batch[0].shape[1]
    sources = dict(zip(algo.SOURCES, batch))
    cost, grads = algo.cost_and_gradients(sources)
    _check_plans(rec, B)
    cost2, again = algo.cost_and_gradients(sources)
    assert cost2 == cost and all(np.array_equal(again[k], g) for k, g in grads.items())
    clean = bench_recognizer()
    clean.set_parameter_values(rec.get_parameter_values())
    assert not np.isclose(cost, clean.cost(*batch).sum() / B, rtol=1e-6, atol=0)     # the noise acted
    for step in range(2):
        algo.process_batch(sources)
        assert np.isfinite(float(algo.last_cost.item())) and np.isfinite(algo.total_gradient_norm()), step
        fresh = bench_recognizer()
        fresh.set_parameter_values(rec.get_parameter_values())
        got, want = rec.cost(*batch), fresh.cost(*batch)
        assert np.array_equal(got, want), (step, float(np.abs(got - want).max()))
        assert rec.launch_status() == (0, 0)
        del fresh
