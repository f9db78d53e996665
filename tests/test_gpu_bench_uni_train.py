"""The forward-only training step tools/bench_unidirectional.py times (bench.NET with bidir False: four forward GRU
layers of 256, encoded width 256), on its whole batch, against float64 gradients: 64 utterances of up to 1500 frames
and 190 label steps with bench.init_values weights, the inputs of bench.train_bench's first shard and its step rule
(bench.TRAIN_CONF, max-norm 1).

tests/golden/make_bench_uni_golden.py builds the gradient as the mean of the gradients of the 64 utterances run one at
a time through tests/unidirectional_oracle.py (exact under the default prior; tests/test_bench_uni_golden_cpu.py checks
that and that the fixture still matches bench.py).  At this size the step runs what no smaller forward-only case
reaches: the taped tensor-core scan in 16 clusters of 4 rows, the projections of layers 1-3 streamed beside the scans
in training, split-K tensor-core weight gradients over 96,000 rows with N = 3 D = 768, and the persistent decoder at
E = 256 with C = 256.  The readout biases are moved off their maxout kinks by the fixture's own offsets.

Bars: those of test_gpu_bench_train.py (its checkers): the cost and the cost matrix to 1e-4, every stored gradient
entry to 1e-4 of its parameter's largest entry plus 1e-6 of the model's, the statistics to 2e-4 of their scale, the
gradient norm to 1e-4, and the parameters after one update against the float64 step rules.  Measured on an H100 80GB
HBM3 (700 W power limit): worst entry error 0.36 of its bar (encoder layer 0), worst statistic 0.37 of its bar, cost
matrix 6.6e-7, gradient norm 209.4495 against 209.4530, parameters after the update 2.3e-3 of their bar; about 2 s
there after the oracle's fixture is loaded."""
import os
import sys
from collections import OrderedDict

import numpy as np
import pytest

import bench
import unidirectional_oracle as U
from helpers import package, rel_err
from oracle import lvsr_oracle_grad as G
from test_gpu_bench_train import TOL, _check_entries, _check_stats, _norm

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _generator():
    if GOLDEN not in sys.path:
        sys.path.insert(0, GOLDEN)
    import make_bench_uni_golden
    return make_bench_uni_golden


def _bench_recognizer(pkg):
    """The forward-only recognizer tools/bench_unidirectional.py trains."""
    W, N = bench.TRAIN_WORKLOAD, bench.NET
    return pkg.SpeechRecognizer(
        input_dims={"recordings": W["F"]}, input_num_chars={}, eos_label=W["V"] - 1, num_phonemes=W["V"],
        dim_dec=N["dim_dec"], dims_bidir=N["dims_bidir"], subsample=N["subsample"], conv_n=N["conv_n"],
        conv_num_filters=N["conv_num_filters"], dim_matcher=N["dim_matcher"], post_merge_dims=N["post_merge_dims"],
        post_merge_activation=pkg.Maxout(2), enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent,
        bidir=False)


def test_forward_only_benchmark_step_matches_float64_gradients(monkeypatch):
    torch = _torch()
    monkeypatch.setenv("LVSR_DEC_CHECK", "1")
    gen = _generator()
    gold = np.load(gen.PATH)
    cfg, batch, params = gen.bench_inputs()
    assert [str(d) for d in gold["batch_sha256"]] == gen.base.batch_digests(batch), "rerun make_bench_uni_golden.py"
    assert str(gold["params_sha256"]) == gen.base.params_digest(params), "rerun make_bench_uni_golden.py"
    params = gen.base.apply_nudges(params, gold["nudge_index"], gold["nudge_value"])
    print("%d maxout units moved off their kinks by at most %.1e: smallest gap %.1e -> %.1e" % (
        gold["nudge_index"].size, np.abs(gold["nudge_value"]).max(), float(gold["min_gap_before"]),
        float(gold["min_gap"])))
    W = bench.TRAIN_WORKLOAD
    B = W["B"]
    pkg = package()
    rec = _bench_recognizer(pkg)
    assert list(rec.parameter_shapes().items()) == list(U.param_shapes(cfg).items())
    rec.set_parameter_values(params)
    sources = dict(zip(pkg.GradientDescent.SOURCES, batch))
    tc = G.make_train_config(max_norm=1.0, **bench.TRAIN_CONF)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(bench.TRAIN_CONF, dict(max_norm=1.0)))
    algo.initialize()

    # ---- cost and gradients of the whole batch
    cost, grads = algo.cost_and_gradients(sources)
    dec_plan, enc_plan, status = rec.decoder_plan(), rec.encoder_plan(), rec.launch_status()
    print("decoder plan:", dec_plan)
    print("encoder plan:", enc_plan)
    want_cost = float(gold["cost"])
    print("cost %.6f (float64 %.6f)" % (cost, want_cost))
    assert abs(cost - want_cost) <= TOL * abs(want_cost)
    worst, bad = _check_entries(gold, grads)
    print("worst entry error / bar per family:", {k: "%.2e" % v for k, v in worst.items()})
    assert not bad, bad
    worst, bad = _check_stats(gen.base, gold, grads)
    print("worst statistic error / bar per family:", {k: "%.2e" % v for k, v in worst.items()})
    assert not bad, bad
    norm = float(gold["grad_norm"])
    print("gradient norm %.6f (float64 %.6f)" % (_norm(grads), norm))
    assert abs(_norm(grads) - norm) <= TOL * norm

    # ---- paths the step ran
    assert status == (0, 0)
    assert dec_plan["ran"] and dec_plan["kernel"].startswith("dec_scan") and dec_plan["nisl"] == B // 16, dec_plan
    frames, T = [], W["T"]
    for k in bench.NET["subsample"]:
        frames.append(T)
        T = -(-T // k)
    assert [p["T"] for p in enc_plan] == frames, enc_plan
    # one direction: ceil(64 / 4) = 16 four-row clusters in one wave
    assert all((p["bigru"], p["rb"], p["clusters"], p["waves"], p["tape"]) == ("mma", 4, 16, 1, True)
               for p in enc_plan), enc_plan
    assert [p["overlap"] for p in enc_plan] == [False, True, True, True], enc_plan
    assert all(p["tiles_beside"] + p["tiles_after"] == -(-p["T"] * B // 128) * 6 for p in enc_plan[1:]), enc_plan
    assert all(p["wgrad"] == "tc" and p["wgrad_splits"] > 1 and p["bwd_cs"] == 8 for p in enc_plan), enc_plan
    assert [p["dx"] for p in enc_plan] == [None] + ["tc"] * 3, enc_plan

    # ---- determinism
    cost2, again = algo.cost_and_gradients(sources)
    assert cost2 == cost
    for k, g in grads.items():
        assert np.array_equal(again[k], g), k

    # ---- the cost matrix of the same forward
    costs = rec.cost(*batch)
    assert rec.launch_status() == (0, 0)
    print("cost matrix rel err %.2e" % rel_err(costs, gold["costs"]))
    assert rel_err(costs, gold["costs"]) < TOL
    assert not costs[batch[3] == 0].any()

    # ---- one update, as bench.train_bench runs it
    p64 = OrderedDict((k, v.astype(np.float64)) for k, v in params.items())
    steps = G.apply_step_rules(p64, OrderedDict((k, g.astype(np.float64)) for k, g in grads.items()), {}, tc)
    algo.process_batch(sources)
    got_norm = algo.total_gradient_norm()
    assert abs(got_norm - norm) <= TOL * norm, (got_norm, norm)
    got = rec.get_parameter_values()
    worst = 0.0
    for k, v in p64.items():
        ref = v - steps[k]
        err = np.abs(got[k] - ref).max()
        bar = 2e-5 * max(1.0, np.abs(ref).max()) + 1e-6
        worst = max(worst, err / bar)
        assert err <= bar, (k, err)
    print("worst parameter error / bar after the update %.2e" % worst)
    torch.cuda.synchronize()
