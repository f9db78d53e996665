"""The training step bench.py --mode train times, on its whole batch, against float64 gradients: 64 utterances of up
to 1500 frames and 190 label steps on the WSJ architecture (bench.NET) with bench.init_values weights, the inputs of
bench.train_bench's first shard and its step rule (bench.TRAIN_CONF, max-norm 1).

The float64 oracle cannot tape this batch, so tests/golden/make_bench_train_golden.py builds its gradient as the mean
of the gradients of the 64 utterances run one at a time (exact under the default prior; tests/test_bench_train_golden_cpu.py
checks that and that the fixture still matches bench.py).  At this size the step runs what smaller tests run as a
trivial case: the persistent decoder's taped forward in four 16-row islands, full 64-row tiles of the decoder's
reverse-time products, the attention backward on 128 CTAs, the tensor-core BiGRU scan and its backward on 64 rows,
float32 sums over R = T*B = 96,000 encoder rows and R = L*B = 12,160 decoder rows, and the update of 5.4 M parameters.
The weights are bench's but for the readout biases the fixture moves by a few 1e-5 to keep every maxout unit off its
kink (make_bench_train_golden.kink_nudges): a float32 forward may take the other piece of a near tie, which moves
that row's whole backward.

Bars: the cost and the cost matrix to 1e-4; every stored gradient entry to helpers.check_grads' bar (1e-4 of the
parameter's largest entry plus 1e-6 of the model's largest); the statistics of every parameter to the bar of
test_gpu_train.py::test_wsj_training_batch_matches_golden_gradients; the gradient norm to 1e-4; the parameters after
each of two updates to train_like_the_oracle's bar against the float64 step rules applied to the GPU's own gradients."""
import importlib.util
import os
import re
from collections import OrderedDict

import numpy as np
import pytest

import bench
from helpers import O, package, rel_err
from oracle import lvsr_oracle_grad as G

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL, ATOL_FRAC, STAT_TOL = 1e-4, 1e-6, 2e-4


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _generator():
    spec = importlib.util.spec_from_file_location("make_bench_train_golden",
                                                  os.path.join(GOLDEN, "make_bench_train_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _bench_recognizer(pkg):
    """The recognizer bench.train_bench builds."""
    W, N = bench.TRAIN_WORKLOAD, bench.NET
    return pkg.SpeechRecognizer(
        input_dims={"recordings": W["F"]}, input_num_chars={}, eos_label=W["V"] - 1, num_phonemes=W["V"],
        dim_dec=N["dim_dec"], dims_bidir=N["dims_bidir"], subsample=N["subsample"], conv_n=N["conv_n"],
        conv_num_filters=N["conv_num_filters"], dim_matcher=N["dim_matcher"], post_merge_dims=N["post_merge_dims"],
        post_merge_activation=pkg.Maxout(2), enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent)


def _family(name):
    if "/encoder/" in name:
        # bidir<l> (Bidirectional layers) or with_fork<l> (forward-only layers)
        return "encoder layer " + re.search(r"/encoder/(?:bidir|with_fork)(\d+)/", name).group(1)
    if name.startswith(O._ATT + "/"):
        return "attention"
    if name.startswith(O._TR + "/"):
        return "transition"
    return "readout and feedback"


def _check_entries(gold, grads):
    """Every stored entry within 1e-4 of its parameter's largest |g| + 1e-6 of the model's; returns the worst
    error / bar per parameter family."""
    names, stats = [str(n) for n in gold["names"]], gold["stats"]
    gmax = stats[:, 2].max()
    worst, bad = {}, []
    for i, k in enumerate(names):
        lo, hi = gold["entry_offsets"][i], gold["entry_offsets"][i + 1]
        idx, want = gold["entry_index"][lo:hi], gold["entry_value"][lo:hi]
        got = grads[k].astype(np.float64).ravel()[idx]
        bar = TOL * stats[i, 2] + ATOL_FRAC * gmax
        e = float(np.abs(got - want).max() / bar)
        f = _family(k)
        worst[f] = max(worst.get(f, 0.0), e)
        if e > 1:
            bad.append((k, e, int(idx[np.argmax(np.abs(got - want))])))
    return worst, bad


def _check_stats(gen, gold, grads):
    """sum, sum |g|, max |g| and the projections at test_wsj_training_batch_matches_golden_gradients' bar: 2e-4 of each
    statistic's natural scale (sum |g| for the sums, max |g| for the maximum, max |g| sqrt(n) for a projection on N(0,1)
    entries); sum g^2 to 2e-4 of itself, as the 1e-4 bar of the gradient norm implies.  Returns the worst error / bar."""
    names, stats = [str(n) for n in gold["names"]], gold["stats"]
    gmax = stats[:, 2].max()
    rng = np.random.RandomState(gen.PROJ_SEED)
    worst, bad = {}, []
    for k, want in zip(names, stats):
        g = grads[k].astype(np.float64)
        r = gen.projections(g.shape, rng)
        got = np.array([g.sum(), np.abs(g).sum(), np.abs(g).max(), (g * g).sum()] +
                       [(g * r[j]).sum() for j in range(gen.NPROJ)])
        scale = np.array([want[1], want[1], want[2], want[3]] + [want[2] * np.sqrt(g.size)] * gen.NPROJ) + ATOL_FRAC * gmax
        e = np.abs(got - want) / scale / STAT_TOL
        f = _family(k)
        worst[f] = max(worst.get(f, 0.0), float(e.max()))
        if e.max() > 1:
            bad.append((k, gen.STAT_NAMES[int(np.argmax(e))], float(e.max())))
    return worst, bad


def _norm(grads):
    return G.l2_norm(grads.values())


def test_benchmarked_training_step_matches_float64_gradients_and_updates(monkeypatch):
    torch = _torch()
    monkeypatch.setenv("LVSR_DEC_CHECK", "1")      # post-condition: launch status 0, no sentinel word left
    gen = _generator()
    gold = np.load(gen.PATH)
    cfg, batch, params = gen.bench_inputs()
    assert [str(d) for d in gold["batch_sha256"]] == gen.batch_digests(batch), "rerun make_bench_train_golden.py"
    assert str(gold["params_sha256"]) == gen.params_digest(params), "rerun make_bench_train_golden.py"
    params = gen.apply_nudges(params, gold["nudge_index"], gold["nudge_value"])
    print("%d maxout units moved off their kinks by at most %.1e: smallest gap %.1e -> %.1e" % (
        gold["nudge_index"].size, np.abs(gold["nudge_value"]).max(), float(gold["min_gap_before"]), float(gold["min_gap"])))
    W = bench.TRAIN_WORKLOAD
    B = W["B"]
    pkg = package()
    rec = _bench_recognizer(pkg)
    # the parameters bench.init_values(rec.parameter_shapes()) draws are those of the fixture
    assert list(rec.parameter_shapes().items()) == list(O.param_shapes(cfg).items())
    rec.set_parameter_values(params)
    sources = dict(zip(pkg.GradientDescent.SOURCES, batch))
    tc = G.make_train_config(max_norm=1.0, **bench.TRAIN_CONF)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(bench.TRAIN_CONF, dict(max_norm=1.0)))
    algo.initialize()

    # ---- cost and gradients of the whole batch
    cost, grads = algo.cost_and_gradients(sources)
    dec_plan, enc_plan, status = rec.decoder_plan(), rec.encoder_plan(), rec.launch_status()
    print("decoder plan of the taped forward:", dec_plan)
    print("encoder plan:", enc_plan)
    want_cost = float(gold["cost"])
    print("cost %.6f (float64 %.6f)" % (cost, want_cost))
    assert abs(cost - want_cost) <= TOL * abs(want_cost)
    worst, bad = _check_entries(gold, grads)
    print("worst entry error / bar per family:", {k: "%.2e" % v for k, v in worst.items()})
    assert not bad, bad
    worst, bad = _check_stats(gen, gold, grads)
    print("worst statistic error / bar per family:", {k: "%.2e" % v for k, v in worst.items()})
    assert not bad, bad
    norm = float(gold["grad_norm"])
    print("gradient norm %.6f (float64 %.6f)" % (_norm(grads), norm))
    assert abs(_norm(grads) - norm) <= TOL * norm

    # ---- paths the step ran
    assert status == (0, 0)
    # lvsr_train_cost_and_grads runs its teacher-forced forward through lvsr_cost_matrix, which records the plan
    assert dec_plan["ran"] and dec_plan["kernel"].startswith("dec_scan") and dec_plan["nisl"] == B // 16, dec_plan
    frames, T = [], W["T"]
    for k in bench.NET["subsample"]:
        frames.append(T)
        T = -(-T // k)
    assert rec.encoded_length(W["T"]) == T
    assert [p["T"] for p in enc_plan] == frames, enc_plan
    assert all(p["bigru"] == "mma" and p["tape"] for p in enc_plan), enc_plan
    assert all(p["wgrad"] == "tc" and p["wgrad_splits"] > 1 for p in enc_plan), enc_plan
    assert [p["dx"] for p in enc_plan] == [None] + ["tc"] * (len(enc_plan) - 1), enc_plan

    # ---- determinism: the backward's reductions run in a fixed order
    cost2, again = algo.cost_and_gradients(sources)
    assert cost2 == cost
    for k, g in grads.items():
        assert np.array_equal(again[k], g), k

    # ---- the cost matrix of the same forward (the host-buffer cost call runs the encoder and lvsr_cost_matrix)
    costs = rec.cost(*batch)
    assert rec.decoder_plan() == dec_plan and rec.launch_status() == (0, 0)
    print("cost matrix rel err %.2e" % rel_err(costs, gold["costs"]))
    assert rel_err(costs, gold["costs"]) < TOL
    assert not costs[batch[3] == 0].any()

    # ---- two updates, as bench.train_bench runs them
    p64 = OrderedDict((k, v.astype(np.float64)) for k, v in params.items())
    state = {}
    step_grads = grads
    for step in range(2):
        if step == 1:
            # the GPU's gradients at the updated parameters, from a second handle
            rec2 = _bench_recognizer(pkg)
            rec2.set_parameter_values(rec.get_parameter_values())
            algo2 = pkg.GradientDescent(recognizer=rec2, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
            _, step_grads = algo2.cost_and_gradients(sources)
            del algo2, rec2
            p64 = OrderedDict((k, v.astype(np.float64)) for k, v in rec.get_parameter_values().items())
        want_norm = float(gold["grad_norm"]) if step == 0 else _norm(step_grads)
        steps = G.apply_step_rules(p64, OrderedDict((k, g.astype(np.float64)) for k, g in step_grads.items()), state, tc)
        algo.process_batch(sources)
        got_norm = algo.total_gradient_norm()
        print("step %d: gradient norm %.6f (want %.6f), %s" % (
            step, got_norm, want_norm, "clipped to %g" % tc["gradient_threshold"] if want_norm >= tc["gradient_threshold"]
            else "not clipped"))
        assert abs(got_norm - want_norm) <= TOL * want_norm, (step, got_norm, want_norm)
        got = rec.get_parameter_values()
        worst = 0.0
        for k, v in p64.items():
            ref = v - steps[k]
            err = np.abs(got[k] - ref).max()
            bar = 2e-5 * max(1.0, np.abs(ref).max()) + 1e-6
            worst = max(worst, err / bar)
            assert err <= bar, (step, k, err)
        print("step %d: worst parameter error / bar %.2e" % (step, worst))
    for k, v in rec.get_parameter_values().items():
        if G.is_weight(k):
            assert (np.sqrt((v.astype(np.float64) ** 2).sum(axis=0)) <= 1.0 + 1e-5).all(), k
    torch.cuda.synchronize()
