"""Task loss estimation (criterion mse_gain / mse_reward) on the GPU against the float64 oracle of tests/tle_oracle.py:
the reward and gain matrices of the reward kernel (exactly), the cost matrix on both decoder plans, analyze against a
different groundtruth, validation statistics, greedy generation and sampling, beam search, the stacked decoder and a
checkpoint round trip, at the TIMIT iclr_reward architecture and the WSJ model bench.py times."""

import numpy as np
import pytest

import bench
import stack_oracle as SO
import tle_oracle as TO
from helpers import O, SMALL, f32, make_recognizer, package, rel_err

pytestmark = pytest.mark.gpu

# exp/timit/configs/iclr_reward.yaml (over nips_smooth / nips_conv): 3 x BiGRU(256) without subsampling, 63 phonemes
ICLR = dict(num_features=123, dims_bidir=[256, 256, 256], subsample=[1, 1, 1], dim_dec=256, dim_matcher=512,
            conv_n=100, conv_num_filters=10, num_phonemes=63, post_merge_dims=[256], maxout_pieces=2)
MODELS = dict(iclr=ICLR, wsj=bench.NET)


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _tle(cfg, params, name="mse_gain", min_reward=-1.0):
    return make_recognizer(cfg, params, criterion=dict(name=name, min_reward=min_reward))


def _setup(net, seed, B=3, T=40, **kw):
    cfg = O.make_config(**dict(net, **kw))
    params = O.init_params(cfg, seed=seed, scale=10.0)
    batch = O.synthetic_batch(cfg, B=B, T=T, seed=seed + 20)
    return cfg, params, batch


def _p64(params):
    """The parameters as the GPU holds them (float32), in float64 for the oracle."""
    return {k: f32(v) for k, v in params.items()}


def _matrices(rec, g, y):
    torch = _torch()
    lib, h = package()._lib.load(), rec._require_ready()
    g = torch.as_tensor(np.ascontiguousarray(g, dtype=np.int64), device=rec.device)
    y = torch.as_tensor(np.ascontiguousarray(y, dtype=np.int64), device=rec.device)
    L, B = y.shape
    V = rec.net["num_phonemes"]
    rewards = torch.empty((L, B, V), dtype=torch.float32, device=rec.device)
    gains = torch.empty_like(rewards)
    package()._lib.check(lib.lvsr_tle_matrices(h, g.data_ptr(), g.shape[0], y.data_ptr(), L, B, rewards.data_ptr(),
                                                gains.data_ptr(), rec._stream()))
    return rewards.cpu().numpy(), gains.cpu().numpy()


def _handle(V, eos=None):
    cfg = O.make_config(**dict(SMALL, num_phonemes=V, eos_label=V - 1 if eos is None else eos))
    return cfg, _tle(cfg, O.init_params(cfg, seed=3))


def _check_matrices(rec, cfg, g, y):
    got_r, got_g = _matrices(rec, g, y)
    want_r, want_g = TO.reward_op(g, y, cfg["num_phonemes"], cfg["eos_label"])
    np.testing.assert_array_equal(got_r, want_r)
    np.testing.assert_array_equal(got_g, want_g)


def _random_pairs(rng, V, eos, B, Lg, L, p_eos=0.1):
    """Groundtruths ending in eos at random lengths (padded with random symbols after it), predictions with eos at
    random places or none."""
    g = rng.randint(0, V, size=(Lg, B))
    g[g == eos] = (eos + 1) % V
    for b in range(B):
        g[rng.randint(0, Lg), b] = eos
    y = rng.randint(0, V, size=(L, B))
    y[rng.rand(L, B) < p_eos] = eos
    return g, y


@pytest.mark.parametrize("V", [5, 32, 63, 128])
def test_reward_and_gain_matrices_match_the_oracle_exactly(V):
    cfg, rec = _handle(V)
    rng = np.random.RandomState(V)
    _check_matrices(rec, cfg, *_random_pairs(rng, V, V - 1, B=9, Lg=30, L=37))
    _check_matrices(rec, cfg, *_random_pairs(rng, V, V - 1, B=5, Lg=12, L=6, p_eos=0.0))


def test_reward_matrices_at_the_edges():
    """A prediction without eos, eos at step 0, groundtruth and prediction lengths 1 and 300."""
    V, eos = 32, 31
    cfg, rec = _handle(V)
    rng = np.random.RandomState(5)
    y = rng.randint(0, eos, size=(20, 2))                                   # no eos at all
    g = np.array([[3, 3], [eos, eos]])
    _check_matrices(rec, cfg, g, y)
    y0 = y.copy()
    y0[0] = eos                                                             # eos at step 0
    _check_matrices(rec, cfg, g, y0)
    _check_matrices(rec, cfg, np.full((1, 2), eos), y)                      # groundtruth of length 1
    _check_matrices(rec, cfg, g, y[:1])                                     # prediction of length 1
    g300, y300 = _random_pairs(rng, V, eos, B=3, Lg=300, L=300, p_eos=0.0)
    g300[:, :] = np.where(g300 == eos, 0, g300)
    g300[-1] = eos                                                          # groundtruth of 300 symbols
    _check_matrices(rec, cfg, g300, y300)


@pytest.mark.parametrize("B", [1, 2, 33, 64, 129])
def test_reward_matrices_of_ragged_batches(B):
    cfg, rec = _handle(63)
    rng = np.random.RandomState(B)
    _check_matrices(rec, cfg, *_random_pairs(rng, 63, 62, B=B, Lg=25, L=40))


def test_missing_eos_names_the_utterance():
    cfg, rec = _handle(32)
    g = np.zeros((6, 4), dtype=np.int64)
    g[3] = 31
    g[:, 2] = 1                                                             # utterance 2 has no eos
    with pytest.raises(RuntimeError, match="utterance 2 does not end in eos"):
        _matrices(rec, g, g)
    _check_matrices(rec, cfg, np.where(np.arange(4) == 2, 31, g), g)      # the handle stays usable


def _costs_vs_oracle(rec, cfg, params, batch, criterion, stepwise, monkeypatch):
    x, xm, y, ym = batch
    torch = _torch()
    if stepwise:
        monkeypatch.setenv("LVSR_NO_DEC_SCAN", "1")
    att, attm = rec.encode(x, xm)
    got = rec.cost_matrix(y, ym, att, attm).cpu().numpy()
    plan = rec.decoder_plan()
    assert plan["ran"] != stepwise
    p, b = _p64(params), [f32(a) if a.dtype != np.int64 else a for a in batch]
    a64, am64 = O.encoder(cfg, p, b[0], b[1])
    want = TO.cost_matrix(cfg, p, a64, am64, y, ym, criterion)
    assert rel_err(got, want) < 2e-4, rel_err(got, want)
    assert torch.isfinite(torch.as_tensor(got)).all()
    return got, want


@pytest.mark.parametrize("model", sorted(MODELS))
@pytest.mark.parametrize("name", ["mse_gain", "mse_reward"])
@pytest.mark.parametrize("min_reward", [-1.0, -5.0])
@pytest.mark.parametrize("stepwise", [False, True])
def test_cost_matrix_matches_the_oracle(model, name, min_reward, stepwise, monkeypatch):
    cfg, params, batch = _setup(MODELS[model], seed=11, B=3, T=40)
    crit = dict(name=name, min_reward=min_reward)
    rec = _tle(cfg, params, name, min_reward)
    _costs_vs_oracle(rec, cfg, params, batch, crit, stepwise, monkeypatch)


@pytest.mark.parametrize("name", ["mse_gain", "mse_reward"])
def test_analyze_scores_the_prediction_against_the_groundtruth(name):
    cfg, params, batch = _setup(ICLR, seed=13, B=1, T=40)
    rec = _tle(cfg, params, name, -5.0)
    x = batch[0][:, 0]
    eos = cfg["eos_label"]
    g = np.array([3, 7, 9, 12, eos], dtype=np.int64)
    pred = np.array([3, 9, 9, eos, 5, 6], dtype=np.int64)
    got = rec.analyze({"recordings": x}, g, pred)[0]
    p = _p64(params)
    a64, am64 = O.encoder(cfg, p, f32(x)[:, None], np.ones((x.shape[0], 1)))
    want = TO.cost_matrix(cfg, p, a64, am64, pred[:, None], None, dict(name=name, min_reward=-5.0),
                          groundtruth=g[:, None])[:, 0]
    assert rel_err(got, want) < 2e-4
    same = rec.analyze({"recordings": x}, g)[0]                             # prediction = groundtruth
    want_same = TO.cost_matrix(cfg, p, a64, am64, g[:, None], None, dict(name=name, min_reward=-5.0))[:, 0]
    assert rel_err(same, want_same) < 2e-4


def test_validation_statistics_report_the_task_loss():
    cfg, params, batch = _setup(ICLR, seed=17, B=4, T=40)
    rec = _tle(cfg, params, "mse_reward", -1.0)
    stats = rec.validation_statistics(*batch)
    p = _p64(params)
    a64, am64 = O.encoder(cfg, p, f32(batch[0]), f32(batch[1]))
    want = TO.cost_matrix(cfg, p, a64, am64, batch[2], batch[3], dict(name="mse_reward", min_reward=-1.0))
    assert abs(stats["cost"] - want.sum()) <= 2e-4 * abs(want).sum()


def test_greedy_generation_and_sampling_start_from_output_zero():
    cfg, params, batch = _setup(ICLR, seed=19, B=2, T=30)
    rec = _tle(cfg, params)
    x, xm = batch[0], batch[1]
    st = rec._initial_states(5, 3)
    assert (st["outputs"].cpu().numpy() == 0).all()
    got = rec.generate(x, xm, n_steps=8, sample=False)
    p = _p64(params)
    a64, am64 = O.encoder(cfg, p, f32(x), f32(xm))
    outs, costs, _ = TO.generate_greedy(cfg, p, a64, am64, 8)
    np.testing.assert_array_equal(got["outputs"], outs)
    assert rel_err(got["costs"], costs) < 1e-4
    sampled = rec.generate(x, xm, n_steps=8, sample=True, seed=7)         # RewardRegressionEmitter.emit is greedy
    np.testing.assert_array_equal(sampled["outputs"], outs)
    np.testing.assert_array_equal(rec.sample({"recordings": x[:, 0]}, n_steps=8)[:, 0],
                                  rec.generate(x[:, :1], None, n_steps=8, sample=False)["outputs"][:, 0])


@pytest.mark.parametrize("beam", [1, 10, 200])
@pytest.mark.parametrize("stop_on", ["patience", "optimistic_future_cost"])
def test_beam_search_on_the_emitter_costs(beam, stop_on):
    cfg, params, batch = _setup(dict(SMALL, num_phonemes=63), seed=23, B=1, T=24)
    bias = params["/recognizer/generator/readout/post_merge/mlp/linear_0.b"]
    bias[:] = -1.0                                      # iclr_reward's readout bias
    bias[cfg["eos_label"]] = -0.6                       # every beam finds hypotheses of one and two symbols
    rec = _tle(cfg, params, "mse_gain", -5.0)
    x = batch[0][:, 0]
    rec.init_beam_search(beam)
    outs, costs = rec.beam_search({"recordings": x}, round_to_inf=4.5, stop_on=stop_on)
    want_outs, want_costs = TO.beam_search(cfg, _p64(params), f32(x), beam, round_to_inf=4.5, stop_on=stop_on)
    assert [list(o) for o in outs[:3]] == want_outs[:3]
    assert rel_err(costs[:3], want_costs[:3]) < 1e-4


def test_stacked_decoder_with_task_loss(monkeypatch):
    cfg = SO.make_config(**SMALL)
    params = SO.init_params(cfg, seed=29, scale=10.0)
    batch = O.synthetic_batch(cfg, B=3, T=30, seed=49)
    rec = _tle(cfg, params, "mse_reward", -1.0)
    x, xm, y, ym = batch
    att, attm = rec.encode(x, xm)
    got = rec.cost_matrix(y, ym, att, attm).cpu().numpy()
    p = _p64(params)
    r = SO.recognizer_cost(cfg, p, f32(x), f32(xm), y, f32(ym), return_all=True)
    ro = O.readout(cfg, SO.wide_params(cfg, p), r["states"], r["weighted_averages"])
    rw, gn = TO.reward_op(y, y, cfg["num_phonemes"], cfg["eos_label"])
    want = TO.tle_cost("mse_reward", ro, y, rw, gn, -1.0, f32(ym))
    assert rel_err(got, want) < 2e-4


def test_checkpoint_round_trip_keeps_the_costs(tmp_path):
    import pickle
    cfg, params, batch = _setup(ICLR, seed=31, B=2, T=30)
    rec = _tle(cfg, params, "mse_gain", -5.0)
    before = rec.cost(*batch)
    path = str(tmp_path / "tle.tar")
    rec.save_params(path)
    other = _tle(cfg, None, "mse_gain", -5.0)
    other.initialize()
    other.load_params(path)
    np.testing.assert_array_equal(other.cost(*batch), before)
    clone = pickle.loads(pickle.dumps(rec))
    assert clone.criterion == dict(name="mse_gain", min_reward=-5.0)
    np.testing.assert_array_equal(clone.cost(*batch), before)
