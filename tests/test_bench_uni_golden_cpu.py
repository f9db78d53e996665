"""The fixture of the forward-only benchmark step (tests/golden/bench_uni_golden.npz, made by
tests/golden/make_bench_uni_golden.py), and the forward-only oracles it and the GPU tests rest on, without a GPU:

- the fixture still describes the batch, weights and configuration tools/bench_unidirectional.py trains
  (bench.NET with bidir False, bench.init_values, the first shard of bench.TRAIN_WORKLOAD);
- its premise holds for one direction: the batch gradient of tests/unidirectional_oracle.py is the mean of the
  gradients of the utterances cropped to their own frames and labels (a padded frame leaves the forward state as it was);
- its kink offsets and its stored entries and statistics are what the generator's rules give;
- tests/bottom_oracle.py composed with the forward-only encoder (cfg["bidir"] False) is the bottom in front of
  unidirectional_oracle's model."""
import json
import os
import sys

import numpy as np
import pytest

import bench
import bottom_oracle as BO
import unidirectional_oracle as U
from helpers import O, PYRAMID

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RERUN = "the forward-only benchmark step changed: rerun python tests/golden/make_bench_uni_golden.py"

if GOLDEN not in sys.path:
    sys.path.insert(0, GOLDEN)
import make_bench_uni_golden as gen  # noqa: E402

base = gen.base


@pytest.fixture(scope="module")
def gold():
    return np.load(gen.PATH)


# ---- the fixture still describes what tools/bench_unidirectional.py trains ---------------------------------------

def test_fixture_matches_the_forward_only_benchmark_step(gold):
    assert json.loads(str(gold["meta"])) == json.loads(json.dumps(gen.meta())), RERUN
    assert gen.SEED == bench.shard_seed(0, base=4321) and gen.NET["bidir"] is False
    cfg, batch, params = gen.bench_inputs()
    assert cfg["bidir"] is False and cfg["dims_bidir"] == bench.NET["dims_bidir"]
    assert [str(d) for d in gold["batch_sha256"]] == base.batch_digests(batch), RERUN
    assert str(gold["params_sha256"]) == base.params_digest(params), RERUN
    assert [str(n) for n in gold["names"]] == list(U.param_shapes(cfg)), RERUN
    assert any("/encoder/with_fork3/" in str(n) for n in gold["names"])
    assert not any("/encoder/bidir" in str(n) for n in gold["names"])
    L, B = batch[2].shape
    assert gold["costs"].shape == (L, B) == (bench.TRAIN_WORKLOAD["L"], bench.TRAIN_WORKLOAD["B"])


# ---- the premise with one direction -----------------------------------------------------------------------------

def _ragged_batch(cfg, lens, label_lens, seed):
    rng = np.random.RandomState(seed)
    T, L, B = max(lens), max(label_lens), len(lens)
    V = cfg["num_phonemes"]
    m = (np.arange(T)[:, None] < np.array(lens)[None, :]).astype(np.float64)
    x = rng.normal(size=(T, B, cfg["num_features"])) * m[:, :, None]
    labels = np.zeros((L, B), dtype=np.int64)
    lm = np.zeros((L, B))
    for b, n in enumerate(label_lens):
        labels[:n - 1, b] = rng.randint(0, V - 1, size=n - 1)
        labels[n - 1, b] = cfg["eos_label"]
        lm[:n, b] = 1
    return x, m, labels, lm


NARROW_BENCH = dict(bench.NET, dims_bidir=[64] * 4, dim_dec=64, dim_matcher=64, post_merge_dims=[64])
CASES = {
    # odd lengths under subsample [1, 2, 2]: 37 -> 19 -> 10, 29 -> 15 -> 8; one utterance of one label
    "pyramid": (PYRAMID, [37, 40, 29, 33], [5, 1, 4, 6]),
    # bench.NET's layers, subsampling and conv_n = 100, narrowed to width 64; the longest utterance is not the first
    "bench_layout": (NARROW_BENCH, [45, 60, 51], [4, 8, 1]),
}


@pytest.mark.parametrize("case", list(CASES))
def test_batch_gradient_is_the_mean_of_cropped_utterance_gradients(case):
    net, lens, label_lens = CASES[case]
    cfg = U.make_config(**net)
    params = U.init_params(cfg, seed=5, scale=10.0)
    batch = _ragged_batch(cfg, lens, label_lens, seed=3)
    cost, grads, costs = U.cost_and_grads(cfg, params, *batch, return_costs=True)
    mcost, mcosts, mgrads = base.mean_of_utterance_grads(cfg, params, batch, oracle=gen.ORACLE)
    assert list(mgrads) == list(grads) == list(U.param_shapes(cfg))
    gmax = max(np.abs(g).max() for g in grads.values())
    worst = 0.0
    for k, g in grads.items():
        err = np.abs(mgrads[k] - g).max() / max(np.abs(g).max(), 1e-3 * gmax)
        worst = max(worst, err)
        assert err < 1e-12, (k, err)
    assert abs(mcost - cost) <= 1e-12 * abs(cost)
    assert np.abs(mcosts - costs).max() <= 1e-12 * np.abs(costs).max()
    assert not mcosts[batch[3] == 0].any()
    print("%s: worst relative difference %.1e" % (case, worst))


def test_generator_refuses_a_window_prior():
    cfg = U.make_config(prior=dict(type="window_around_median", before=5, after=7), **PYRAMID)
    params = U.init_params(cfg, seed=5, scale=10.0)
    batch = _ragged_batch(cfg, [37, 40], [5, 1], seed=3)
    with pytest.raises(ValueError, match="default prior"):
        base.mean_of_utterance_grads(cfg, params, batch, oracle=gen.ORACLE)


# ---- the fixture agrees with the generator's rules ----------------------------------------------------------------

def test_fixture_kink_offsets(gold):
    eps = float(gold["kink_eps"])
    assert eps == base.KINK_EPS
    idx, val = gold["nudge_index"], gold["nudge_value"]
    cfg, _, params = gen.bench_inputs()
    bias = params["/recognizer/generator/readout/post_merge/bias.b"]
    assert idx.size > 0 and np.unique(idx).size == idx.size and (idx % cfg["maxout_pieces"] == 0).all()
    assert idx.max() < bias.size and not bias[idx].any()
    assert val.dtype == np.float32 and (np.abs(val) > 0).all() and (np.abs(val) <= 100 * eps).all()
    assert float(gold["min_gap_before"]) < eps <= float(gold["min_gap"])
    moved = base.apply_nudges(params, idx, val)
    assert [k for k in params if not np.array_equal(params[k], moved[k])] == [
        "/recognizer/generator/readout/post_merge/bias.b"]


def test_fixture_is_self_consistent(gold):
    cfg, batch, _ = gen.bench_inputs()
    shapes = U.param_shapes(cfg)
    names, stats = [str(n) for n in gold["names"]], gold["stats"]
    assert stats.shape == (len(names), len(base.STAT_NAMES))
    assert gold["entry_offsets"][-1] == gold["entry_index"].size == gold["entry_value"].size
    rng = np.random.RandomState(base.PROJ_SEED)
    for i, k in enumerate(names):
        shape = shapes[k]
        size = int(np.prod(shape))
        lo, hi = gold["entry_offsets"][i], gold["entry_offsets"][i + 1]
        idx, val = gold["entry_index"][lo:hi], gold["entry_value"][lo:hi]
        r = base.projections(shape, rng)
        assert idx.min() >= 0 and idx.max() < size and np.unique(idx).size == idx.size, k
        if size <= base.FULL_MAX:
            assert np.array_equal(idx, np.arange(size)), k
            g = val.reshape(shape)
            want = np.array([g.sum(), np.abs(g).sum(), np.abs(g).max(), (g * g).sum()] +
                            [(g * r[j]).sum() for j in range(base.NPROJ)])
            assert np.allclose(stats[i], want, rtol=1e-12, atol=1e-15 * stats[i, 1]), k
        else:
            assert idx.size == base.TOP + base.SAMPLED, k
            top, rest = np.abs(val[:base.TOP]), np.abs(val[base.TOP:])
            assert top.max() == stats[i, 2] and top.min() >= rest.max(), k
        assert 0 < stats[i, 2] <= stats[i, 1] and abs(stats[i, 0]) <= stats[i, 1], k
    assert np.isclose(np.sqrt(stats[:, 3].sum()), float(gold["grad_norm"]), rtol=1e-12)
    costs, lm = gold["costs"], batch[3]
    assert not costs[lm == 0].any() and (costs[lm > 0] > 0).all()
    assert np.isclose(costs.sum() / costs.shape[1], float(gold["cost"]), rtol=1e-12)
    assert os.path.getsize(gen.PATH) < 1 << 20


# ---- bottom_oracle composed with the forward-only encoder ---------------------------------------------------------

def _bottom_config(activation="relu"):
    return BO.make_config(U.make_config(**dict(PYRAMID, dims_bidir=[64, 128], subsample=[1, 2])), [48, 40],
                          activation)


def test_bottom_composition_parameter_table():
    """The forward-only table of the inner model (num_features = the bottom's last width) with the bottom's
    linears after the encoder's with_fork layers and before the generator's."""
    cfg = _bottom_config()
    names = list(BO.param_shapes(cfg))
    inner = list(U.param_shapes(BO.inner(cfg)))
    bottom = [BO.linear_name(i) + s for i in range(2) for s in (".W", ".b")]
    n_enc = sum(1 for k in inner if k.startswith(U.ENC + "/"))
    assert n_enc == 14 and names == inner[:n_enc] + bottom + inner[n_enc:]
    assert BO.param_shapes(cfg)[U.layer_base(0) + "/fork/fork_inputs.W"] == (40, 64)
    assert BO.param_shapes(cfg)[BO.linear_name(0) + ".W"] == (PYRAMID["num_features"], 48)


@pytest.mark.parametrize("attention", ["content_and_conv", "content"])
def test_bottom_composition_is_the_inner_model_on_bottom_features(attention):
    """An identity bottom (one Rectifier layer, W = I, b = 0, positive features) leaves the recordings as they are: the
    composed cost, encoder and gradients of every inner parameter are unidirectional_oracle's own; a general bottom
    gives U's cost on bottom(recordings), and its float64 mirror agrees with the numpy cost."""
    F = PYRAMID["num_features"]
    cfg = BO.make_config(U.make_config(attention_type=attention, **dict(PYRAMID, dims_bidir=[64, 128],
                                                                         subsample=[1, 2])), [F], "relu")
    params = BO.init_params(cfg, seed=7, scale=10.0)
    params[BO.linear_name(0) + ".W"] = np.eye(F)
    params[BO.linear_name(0) + ".b"] = np.zeros(F)
    x, m, labels, lm = _ragged_batch(cfg, [23, 17, 20], [4, 2, 3], seed=9)
    x = np.abs(x) + 0.1 * m[:, :, None]
    inner = BO.inner(cfg)
    ip = {k: v for k, v in params.items() if not k.startswith(BO.BOTTOM)}
    assert np.array_equal(BO.encoder(cfg, params, x, m)[0], U.encoder(inner, ip, x, m)[0])
    want = U.recognizer_cost(inner, ip, x, m, labels, lm)
    assert np.allclose(BO.recognizer_cost(cfg, params, x, m, labels, lm), want, rtol=1e-13, atol=0)
    cost, grads = BO.cost_and_grads(cfg, params, x, m, labels, lm)
    icost, igrads = U.cost_and_grads(inner, ip, x, m, labels, lm)
    assert abs(cost - icost) <= 1e-12 * abs(icost) and abs(cost - want.sum() / 3) <= 1e-10 * abs(cost)
    for k, g in igrads.items():
        assert np.allclose(grads[k], g, rtol=1e-10, atol=1e-12 * np.abs(g).max()), k
    assert np.abs(grads[BO.linear_name(0) + ".W"]).max() > 0

    params = BO.init_params(cfg, seed=8, scale=10.0)
    params[BO.linear_name(0) + ".b"] = np.random.RandomState(1).normal(0, 0.3, size=F)
    feats = BO.bottom(cfg, params, x)
    assert not np.array_equal(feats, x)
    want = U.recognizer_cost(inner, params, feats, m, labels, lm)
    got = BO.recognizer_cost(cfg, params, x, m, labels, lm)
    assert np.allclose(got, want, rtol=1e-13, atol=0)
    cost, _ = BO.cost_and_grads(cfg, params, x, m, labels, lm)
    assert abs(cost - got.sum() / 3) <= 1e-10 * abs(cost)


def test_bottom_composition_gradient_against_finite_differences():
    """Central differences of the composed cost in one entry of each bottom layer (Tanh: no kink for a difference to
    straddle) and of the forward-only layer 0."""
    cfg = _bottom_config("tanh")
    params = BO.init_params(cfg, seed=11, scale=10.0)
    rng = np.random.RandomState(12)
    for i in range(2):
        params[BO.linear_name(i) + ".b"] = rng.normal(0, 0.3, size=params[BO.linear_name(i) + ".b"].shape)
    x, m, labels, lm = _ragged_batch(cfg, [15, 12], [3, 2], seed=13)
    _, grads = BO.cost_and_grads(cfg, params, x, m, labels, lm)
    for k, idx in ((BO.linear_name(0) + ".W", (3, 5)), (BO.linear_name(1) + ".W", (7, 2)),
                   (U.layer_base(0) + "/fork/fork_gate_inputs.W", (4, 9))):
        h = 1e-6
        vals = []
        for s in (h, -h):
            p = dict(params)
            p[k] = params[k].copy()
            p[k][idx] += s
            vals.append(BO.recognizer_cost(cfg, p, x, m, labels, lm).sum() / 2)
        fd = (vals[0] - vals[1]) / (2 * h)
        assert abs(fd - grads[k][idx]) <= 1e-6 * max(1.0, abs(fd)), (k, fd, grads[k][idx])
