"""The fixture of the benchmarked training step (tests/golden/bench_train_golden.npz, made by
tests/golden/make_bench_train_golden.py), without a GPU:

- it still describes the batch, weights and configuration bench.py --mode train times;
- its premise holds: under the default prior the batch gradient of the float64 oracle is the mean of the gradients of
  the utterances cropped to their own frames and labels, and the generator refuses a window prior, for which it is not;
- the readout bias offsets that keep the maxout units off their kinks are small and clear every row;
- its stored entries and statistics agree with each other."""
import importlib.util
import json
import os

import numpy as np
import pytest

import bench
from helpers import O, PYRAMID
from oracle import lvsr_oracle_grad as G

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RERUN = "the benchmark's training step changed: rerun python tests/golden/make_bench_train_golden.py"


def _generator():
    spec = importlib.util.spec_from_file_location("make_bench_train_golden",
                                                  os.path.join(GOLDEN, "make_bench_train_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


gen = _generator()


@pytest.fixture(scope="module")
def gold():
    return np.load(gen.PATH)


# ---- the fixture still describes what bench.py times ------------------------------------------------------------

def test_fixture_matches_the_benchmarked_training_step(gold):
    """Workload, net, step rules and seed as bench.py has them, and inputs and initial weights that hash to the
    fixture's digests, so a change of the benchmark fails here instead of comparing against stale numbers."""
    assert json.loads(str(gold["meta"])) == json.loads(json.dumps(gen.meta())), RERUN
    assert gen.SEED == bench.shard_seed(0, base=4321)
    cfg, batch, params = gen.bench_inputs()
    assert [str(d) for d in gold["batch_sha256"]] == gen.batch_digests(batch), RERUN
    assert str(gold["params_sha256"]) == gen.params_digest(params), RERUN
    assert [str(n) for n in gold["names"]] == list(O.param_shapes(cfg)), RERUN
    L, B = batch[2].shape
    assert gold["costs"].shape == (L, B) == (bench.TRAIN_WORKLOAD["L"], bench.TRAIN_WORKLOAD["B"])


def test_digests_see_every_input():
    """One changed value of any input or weight changes its digest."""
    _, batch, params = gen.bench_inputs()
    ref = gen.batch_digests(batch)
    for i in range(4):
        b = [a.copy() for a in batch]
        b[i].flat[b[i].size // 2] += 1
        assert gen.batch_digests(b)[i] != ref[i]
    p = dict(params)
    k = list(p)[-1]
    p[k] = p[k].copy()
    p[k].flat[0] = np.nextafter(p[k].flat[0], np.float32(1))
    assert gen.params_digest(p) != gen.params_digest(params)


# ---- the premise: the batch gradient is the mean of per-utterance gradients -------------------------------------

def _ragged_batch(cfg, lens, label_lens, seed):
    """Right-padded batch of utterances of the given frame and label counts (eos last), N(0,1) features."""
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
    # odd lengths under subsample [1, 2, 2]: 37 -> 19 -> 10, 29 -> 15 -> 8, 33 -> 17 -> 9; one utterance of one label
    "pyramid": (PYRAMID, [37, 40, 29, 33], [5, 1, 4, 6]),
    # bench.NET's layers, subsampling and conv_n = 100, narrowed to width 64; the longest utterance is not the first
    "bench_layout": (NARROW_BENCH, [45, 60, 51], [4, 8, 1]),
}


@pytest.mark.parametrize("case", list(CASES))
def test_batch_gradient_is_the_mean_of_cropped_utterance_gradients(case):
    net, lens, label_lens = CASES[case]
    cfg = O.make_config(**net)
    params = O.init_params(cfg, seed=5, scale=10.0)
    batch = _ragged_batch(cfg, lens, label_lens, seed=3)
    assert [int(v) for v in batch[1].sum(0)] == lens and [int(v) for v in batch[3].sum(0)] == label_lens
    cost, grads, costs = G.cost_and_grads(cfg, params, *batch, return_costs=True)
    mcost, mcosts, mgrads = gen.mean_of_utterance_grads(cfg, params, batch)
    assert list(mgrads) == list(grads)
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


@pytest.mark.parametrize("prior", [dict(type="window_around_median", before=5, after=7),
                                   dict(type="window_around_mean", before=5, after=7),
                                   dict(type="expanding", initial_begin=0, initial_end=6, min_speed=0.7, max_speed=2.2)],
                         ids=lambda p: p["type"])
def test_generator_refuses_a_window_prior(prior, monkeypatch):
    """A window prior cuts one window for the whole batch, so an utterance's gradient depends on the others'."""
    cfg = O.make_config(prior=prior, **PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    batch = _ragged_batch(cfg, [37, 40], [5, 1], seed=3)
    monkeypatch.setattr(G, "cost_and_grads", lambda *a, **k: pytest.fail("the oracle ran"))
    with pytest.raises(ValueError, match="default prior"):
        gen.mean_of_utterance_grads(cfg, params, batch)


# ---- maxout kinks ------------------------------------------------------------------------------------------------

def test_kink_nudges_clear_every_row_of_a_unit():
    eps = gen.KINK_EPS
    rng = np.random.RandomState(0)
    gaps = rng.uniform(0.5, 1.0, size=(50, 6)) * rng.choice([-1, 1], size=(50, 6))
    gaps[3, 1] = 1e-7                  # a near tie
    gaps[7, 1] = -1.2 * eps            # a positive offset has to jump over this row: at least 2.2 eps
    gaps[9, 4] = -0.4 * eps
    nudges = gen.kink_nudges(gaps)
    assert sorted(nudges) == [1, 4]
    for j, d in nudges.items():
        assert np.abs(gaps[:, j] + float(d)).min() >= eps
    # the smallest multiples of eps / 4 that clear every row of the unit
    assert float(nudges[1]) == pytest.approx(-1.25 * eps) and float(nudges[4]) == pytest.approx(-0.75 * eps)


def test_fixture_kink_offsets(gold):
    """The fixture's offsets move only zero biases of first maxout pieces, by a few KINK_EPS, and leave every
    label-unmasked row at least KINK_EPS from its kink where bench's weights had rows closer than that."""
    eps = float(gold["kink_eps"])
    assert eps == gen.KINK_EPS
    idx, val = gold["nudge_index"], gold["nudge_value"]
    cfg, _, params = gen.bench_inputs()
    bias = params["/recognizer/generator/readout/post_merge/bias.b"]
    assert idx.size > 0 and np.unique(idx).size == idx.size and (idx % cfg["maxout_pieces"] == 0).all()
    assert idx.max() < bias.size and not bias[idx].any()
    assert val.dtype == np.float32 and (np.abs(val) > 0).all() and (np.abs(val) <= 100 * eps).all()
    assert float(gold["min_gap_before"]) < eps <= float(gold["min_gap"])
    moved = gen.apply_nudges(params, idx, val)
    assert [k for k in params if not np.array_equal(params[k], moved[k])] == ["/recognizer/generator/readout/post_merge/bias.b"]


# ---- the fixture agrees with itself ------------------------------------------------------------------------------

def _entries(gold, i):
    lo, hi = gold["entry_offsets"][i], gold["entry_offsets"][i + 1]
    return gold["entry_index"][lo:hi], gold["entry_value"][lo:hi]


def test_fixture_is_self_consistent(gold):
    cfg = O.make_config(**bench.NET)
    shapes = O.param_shapes(cfg)
    names, stats = [str(n) for n in gold["names"]], gold["stats"]
    assert stats.shape == (len(names), len(gen.STAT_NAMES))
    assert gold["entry_offsets"][-1] == gold["entry_index"].size == gold["entry_value"].size
    rng = np.random.RandomState(gen.PROJ_SEED)
    full = 0
    for i, k in enumerate(names):
        shape = shapes[k]
        size = int(np.prod(shape))
        idx, val = _entries(gold, i)
        r = gen.projections(shape, rng)                     # drawn for every parameter, in order
        assert idx.min() >= 0 and idx.max() < size and np.unique(idx).size == idx.size, k
        if size <= gen.FULL_MAX:
            full += 1
            assert np.array_equal(idx, np.arange(size)), k
            g = val.reshape(shape)
            want = np.array([g.sum(), np.abs(g).sum(), np.abs(g).max(), (g * g).sum()] +
                            [(g * r[j]).sum() for j in range(gen.NPROJ)])
            assert np.allclose(stats[i], want, rtol=1e-12, atol=1e-15 * stats[i, 1]), k
        else:
            assert idx.size == gen.TOP + gen.SAMPLED, k
            top, rest = np.abs(val[:gen.TOP]), np.abs(val[gen.TOP:])
            assert top.max() == stats[i, 2] and top.min() >= rest.max(), k
            assert (top ** 2).sum() <= stats[i, 3] * (1 + 1e-12), k
        assert 0 < stats[i, 2] <= stats[i, 1] and abs(stats[i, 0]) <= stats[i, 1], k
    assert full == 33 and sum(int(np.prod(shapes[k])) for k in names if np.prod(shapes[k]) <= gen.FULL_MAX) == 16634
    assert np.isclose(np.sqrt(stats[:, 3].sum()), float(gold["grad_norm"]), rtol=1e-12)
    _, batch, _ = gen.bench_inputs()
    costs, lm = gold["costs"], batch[3]
    assert not costs[lm == 0].any() and (costs[lm > 0] > 0).all()
    assert np.isclose(costs.sum() / costs.shape[1], float(gold["cost"]), rtol=1e-12)
    assert os.path.getsize(gen.PATH) < 1 << 20
