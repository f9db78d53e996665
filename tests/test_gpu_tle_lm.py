"""Task loss estimation with an FST language model (criterion mse_gain / mse_reward with net.lm) on the GPU against the
float64 oracle of tests/tle_lm_oracle.py: the loss of the fused readouts on both decoder plans and in analyze, every
normalisation setting, the emitter's fused rows, greedy generation and sampling with the LM state carried, beam search
one utterance at a time and batched, the stacked decoder, a deep readout, content attention, vocabulary widths, a
non-default stream, the training refusal, the weight-0 identity, and compat's search with decode_tle.sh's overrides."""
import os
import pickle
import sys

import numpy as np
import pytest

import content_oracle as CO
import lm_oracle as LO
import readout_oracle as RO
import stack_oracle as SO
import tle_lm_oracle as TLO
from helpers import O, SMALL, f32, make_recognizer, package, rel_err

pytestmark = pytest.mark.gpu

# exp/timit/configs/iclr_reward.yaml (over nips_smooth / nips_conv): 3 x BiGRU(256) without subsampling, 63 phonemes
ICLR = dict(num_features=123, dims_bidir=[256, 256, 256], subsample=[1, 1, 1], dim_dec=256, dim_matcher=512,
            conv_n=100, conv_num_filters=10, num_phonemes=63, post_merge_dims=[256], maxout_pieces=2)
FLAGS = [dict(normalize_am_weights=a, normalize_lm_weights=l, normalize_tot_weights=t)
         for a in (True, False) for l in (True, False) for t in (True, False)]
# decode_tle.sh: net.lm.weight 0.15, every other option at the recognizer's default
DECODE_TLE = dict(weight=0.15, normalize_am_weights=True, normalize_lm_weights=False, normalize_tot_weights=False,
                  am_beta=1.0, no_transition_cost=1e12)


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


_FILES = {}


def _lm_file(tmp_path_factory, V):
    if V not in _FILES:
        S, start, arcs = LO.char_ngram(V, seed=7, n_tri=max(4, min(60, V)), dup=min(6, V), dead=2)
        path = str(tmp_path_factory.mktemp("lm%d" % V) / "lm.fst")
        cmap = LO.to_file(path, V, S, start, arcs, seed=2)
        _FILES[V] = (path, cmap, LO.from_tables(package().lm.load(path, cmap, V)))
    return _FILES[V]


@pytest.fixture(scope="module")
def lm_files(tmp_path_factory):
    return lambda V: _lm_file(tmp_path_factory, V)


def _p64(params):
    return {k: f32(v) for k, v in params.items()}


def _rec(cfg, params, lm_file, o, name="mse_gain", min_reward=-1.0):
    path, cmap, _ = lm_file
    return make_recognizer(cfg, params, criterion=dict(name=name, min_reward=min_reward), lm=dict(o, path=path),
                           character_map=cmap)


def _reattach(rec, o):
    """The handle's fusion options replaced in place (set_lm keeps the criterion)."""
    rec.lm.update(o)
    rec._attach_lm(package()._lib.load(), rec._require_ready())


def _setup(net, seed, B=3, T=40, module=O, **kw):
    cfg = module.make_config(**dict(net, **kw))
    params = module.init_params(cfg, seed=seed, scale=10.0)
    batch = O.synthetic_batch(cfg, B=B, T=T, seed=seed + 20)
    return cfg, params, batch


def _attended(cfg, params, x, m):
    return O.encoder(cfg, _p64(params), f32(x), None if m is None else f32(m))


# ---- the cost matrix and analyze ------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["mse_gain", "mse_reward"])
@pytest.mark.parametrize("min_reward", [-1.0, -5.0])
@pytest.mark.parametrize("stepwise", [False, True], ids=["persistent", "stepwise"])
def test_cost_matrix_matches_the_oracle(lm_files, name, min_reward, stepwise, monkeypatch):
    torch = _torch()
    if stepwise:
        monkeypatch.setenv("LVSR_NO_DEC_SCAN", "1")
    cfg, params, (x, xm, y, ym) = _setup(ICLR, seed=11)
    lm = lm_files(63)
    o = dict(DECODE_TLE, weight=0.5, no_transition_cost=20.0)
    rec = _rec(cfg, params, lm, o, name, min_reward)
    att, attm = rec.encode(x, xm)
    got = rec.cost_matrix(y, ym, att, attm).cpu().numpy()
    assert rec.decoder_plan()["ran"] != stepwise
    a64, am64 = _attended(cfg, params, x, xm)
    crit = dict(name=name, min_reward=min_reward)
    want = TLO.cost_matrix(cfg, _p64(params), lm[2], o, a64, am64, y, ym, crit)
    assert rel_err(got, want) < 2e-4, rel_err(got, want)
    assert torch.isfinite(torch.as_tensor(got)).all()
    # the host entry point (cost) takes the same path
    assert rel_err(rec.cost(x, xm, y, ym), want) < 2e-4


@pytest.mark.parametrize("name", ["mse_gain", "mse_reward"])
def test_every_normalisation_am_beta_and_weight(lm_files, name):
    _torch()
    cfg, params, (x, xm, y, ym) = _setup(ICLR, seed=12, B=2, T=30)
    lm = lm_files(63)
    rec = _rec(cfg, params, lm, DECODE_TLE, name, -5.0)
    att, attm = rec.encode(x, xm)
    a64, am64 = _attended(cfg, params, x, xm)
    r = O.cost_matrix(cfg, _p64(params), a64, am64, y, ym, return_all=True)
    logits = O.readout(cfg, _p64(params), r["states"], r["weighted_averages"])
    crit = dict(name=name, min_reward=-5.0)
    n = 0
    for flags in FLAGS:
        for am_beta in (1.0, 0.7):
            for weight in (0.0, 0.15, 0.5, 2.0):
                o = dict(flags, am_beta=am_beta, weight=weight, no_transition_cost=20.0)
                _reattach(rec, o)
                got = rec.cost_matrix(y, ym, att, attm).cpu().numpy()
                want = TLO.cost_of_logits(cfg, lm[2], o, crit, logits, y, ym)
                assert rel_err(got, want) < 2e-4, (o, rel_err(got, want))
                n += 1
    print("settings compared:", n)


@pytest.mark.parametrize("name", ["mse_gain", "mse_reward"])
@pytest.mark.parametrize("stepwise", [False, True], ids=["persistent", "stepwise"])
def test_analyze_scores_the_fused_prediction_against_the_groundtruth(lm_files, name, stepwise, monkeypatch):
    _torch()
    if stepwise:
        monkeypatch.setenv("LVSR_NO_DEC_SCAN", "1")
    cfg, params, batch = _setup(ICLR, seed=13, B=1, T=40)
    lm = lm_files(63)
    o = dict(DECODE_TLE, no_transition_cost=20.0, weight=0.5)
    rec = _rec(cfg, params, lm, o, name, -5.0)
    x = batch[0][:, 0]
    eos = cfg["eos_label"]
    g = np.array([3, 7, 9, 12, eos], dtype=np.int64)
    pred = np.array([3, 9, 9, eos, 5, 6], dtype=np.int64)
    got = rec.analyze({"recordings": x}, g, pred)
    assert rec.decoder_plan()["ran"] != stepwise
    a64, am64 = _attended(cfg, params, x[:, None], np.ones((x.shape[0], 1)))
    crit = dict(name=name, min_reward=-5.0)
    # the LM rows follow the prediction, the rewards compare it with the groundtruth
    want = TLO.cost_matrix(cfg, _p64(params), lm[2], o, a64, am64, pred[:, None], None, crit, groundtruth=g[:, None],
                           return_all=True)
    assert rel_err(got[0], want["costs"][:, 0]) < 2e-4
    assert rel_err(got[1], want["weights"][:, 0]) < 1e-4
    same = rec.analyze({"recordings": x}, g)[0]
    want_same = TLO.cost_matrix(cfg, _p64(params), lm[2], o, a64, am64, g[:, None], None, crit)[:, 0]
    assert rel_err(same, want_same) < 2e-4


def test_weight_zero_without_normalisation_is_the_handle_without_an_lm(lm_files):
    _torch()
    cfg, params, (x, xm, y, ym) = _setup(ICLR, seed=14, B=3, T=30)
    lm = lm_files(63)
    for name in ("mse_gain", "mse_reward"):
        plain = make_recognizer(cfg, params, criterion=dict(name=name, min_reward=-5.0))
        fused = _rec(cfg, params, lm, dict(weight=0.0, am_beta=1.0, normalize_am_weights=False,
                                           normalize_lm_weights=False, normalize_tot_weights=False), name, -5.0)
        np.testing.assert_array_equal(fused.cost(x, xm, y, ym), plain.cost(x, xm, y, ym))
        att, attm = plain.encode(x, xm)
        np.testing.assert_array_equal(fused.cost_matrix(y, ym, att, attm).cpu().numpy(),
                                      plain.cost_matrix(y, ym, att, attm).cpu().numpy())
        a = fused.generate(x, xm, n_steps=6, sample=False)
        b = plain.generate(x, xm, n_steps=6, sample=False)
        np.testing.assert_array_equal(a["outputs"], b["outputs"])
        np.testing.assert_array_equal(a["costs"], b["costs"])


# ---- the emitter's rows, generation and sampling -------------------------------------------------------------

def test_logprob_rows_are_the_fused_emitter_costs(lm_files):
    torch = _torch()
    cfg, params, (x, xm, _, _) = _setup(ICLR, seed=15, B=2, T=30)
    lm = lm_files(63)
    o = dict(DECODE_TLE, weight=0.5, no_transition_cost=20.0, normalize_lm_weights=True)
    rec = _rec(cfg, params, lm, o)
    att, attm = rec.encode(x, xm)
    ctx = dict(attended=att, attended_mask=attm, preprocessed=rec.preprocess(att))
    B, Tp = att.shape[1], att.shape[0]
    st = rec._initial_states(Tp, B)
    st.update(rec._lm_initial_states(B))
    p = _p64(params)
    a64, am64 = _attended(cfg, params, x, xm)
    ost = TLO.initial_states(cfg, p, lm[2], o, B, a64)
    rng = np.random.RandomState(3)
    for step in range(5):
        got = rec._logprobs(ctx, st).cpu().numpy()
        want = TLO.emitter_costs(cfg, p, o, a64, am64, ost)
        assert rel_err(got, want) < 2e-4, (step, rel_err(got, want))
        # without the LM rows the same call gives -r, the task-loss emitter's unfused costs
        bare = rec._logprobs(ctx, {k: v for k, v in st.items() if not k.startswith("lm_")}).cpu().numpy()
        wa, _, _, _ = O.take_glimpses(cfg, p, a64, None, am64, ost["weights"], ost["step"], ost["states"])
        assert rel_err(bare, -O.readout(cfg, p, ost["states"], wa)) < 2e-4
        y = rng.randint(0, cfg["num_phonemes"], size=B)
        lm_st = rec._lm_next_states(st, torch.as_tensor(y, device=rec.device))
        st = rec._next_states(ctx, st, y)
        st.update(lm_st)
        ost = TLO.next_states(cfg, p, lm[2], o, a64, am64, ost, y)


def test_greedy_generation_and_sampling_carry_the_lm(lm_files):
    _torch()
    cfg, params, (x, xm, _, _) = _setup(ICLR, seed=19, B=2, T=30)
    lm = lm_files(63)
    o = dict(DECODE_TLE, weight=0.5, no_transition_cost=20.0)
    rec = _rec(cfg, params, lm, o)
    got = rec.generate(x, xm, n_steps=8, sample=False)
    a64, am64 = _attended(cfg, params, x, xm)
    outs, costs, _ = TLO.generate_greedy(cfg, _p64(params), lm[2], o, a64, am64, 8)
    np.testing.assert_array_equal(got["outputs"], outs)
    assert rel_err(got["costs"], costs) < 1e-4
    plain = make_recognizer(cfg, params, criterion=dict(name="mse_gain"))
    assert not np.array_equal(plain.generate(x, xm, n_steps=8, sample=False)["outputs"], outs)   # the LM steers
    sampled = rec.generate(x, xm, n_steps=8, sample=True, seed=7)      # RewardRegressionEmitter.emit is greedy
    np.testing.assert_array_equal(sampled["outputs"], outs)
    np.testing.assert_array_equal(rec.sample({"recordings": x[:, 0]}, n_steps=8)[:, 0],
                                  rec.generate(x[:, :1], None, n_steps=8, sample=False)["outputs"][:, 0])


# ---- beam search ---------------------------------------------------------------------------------------------

def _search_model(seed=23, V=63):
    cfg, params, _ = _setup(dict(SMALL, num_phonemes=V), seed=seed, B=1, T=24)
    bias = params["/recognizer/generator/readout/post_merge/mlp/linear_0.b"]
    bias[:] = -1.0                                      # iclr_reward's readout bias
    bias[cfg["eos_label"]] = 1.0                        # eos outweighs the LM's costs: beam 1 finishes too
    return cfg, params


@pytest.mark.parametrize("beam", [1, 10, 200])
@pytest.mark.parametrize("stop_on", ["patience", "optimistic_future_cost"])
def test_beam_search_matches_the_oracle(lm_files, beam, stop_on):
    _torch()
    cfg, params = _search_model()
    lm = lm_files(63)
    # the readouts unnormalised, as the task-loss emitter sees them, plus half the LM's costs
    o = dict(DECODE_TLE, weight=0.5, no_transition_cost=20.0, normalize_am_weights=False)
    rec = _rec(cfg, params, lm, o, "mse_gain", -5.0)
    rng = np.random.RandomState(5)
    utts = [rng.normal(size=(T, cfg["num_features"])).astype(np.float32) for T in (24, 17, 30)]
    rec.init_beam_search(beam)
    batched = rec._beam_search.search_many(utts, cfg["eos_label"], [int(u.shape[0] / cfg["max_decoded_length_scale"])
                                                                    for u in utts],
                                           stop_on=stop_on, raise_on_failure=False)
    n = 0
    for u, b in zip(utts, batched):
        try:
            want_outs, want_costs = TLO.beam_search(cfg, _p64(params), lm[2], o, f32(u), beam, stop_on=stop_on)
        except O.CandidateNotFoundError:
            assert b is None
            with pytest.raises(package().CandidateNotFoundError):
                rec.beam_search({"recordings": u}, stop_on=stop_on)
            continue
        single = rec.beam_search({"recordings": u}, stop_on=stop_on)
        for got_outs, got_costs in (single, b):
            k = min(3, len(want_outs))
            assert [list(t) for t in got_outs[:k]] == want_outs[:k]
            assert rel_err(got_costs[:k], want_costs[:k]) < 1e-4
        n += len(want_outs)
    print("finished hypotheses of the oracle:", n)
    assert n >= 1


# ---- the model variants ----------------------------------------------------------------------------------------

def test_stacked_decoder(lm_files, monkeypatch):
    _torch()
    cfg = SO.make_config(**SMALL)
    params = SO.init_params(cfg, seed=29, scale=10.0)
    x, xm, y, ym = O.synthetic_batch(cfg, B=3, T=30, seed=49)
    lm = lm_files(cfg["num_phonemes"])
    o = dict(DECODE_TLE, weight=0.5, no_transition_cost=20.0)
    rec = _rec(cfg, params, lm, o, "mse_reward", -1.0)
    got = rec.cost(x, xm, y, ym)
    p = _p64(params)
    r = SO.recognizer_cost(cfg, p, f32(x), f32(xm), y, f32(ym), return_all=True)
    logits = O.readout(cfg, SO.wide_params(cfg, p), r["states"], r["weighted_averages"])
    want = TLO.cost_of_logits(cfg, lm[2], o, dict(name="mse_reward", min_reward=-1.0), logits, y, f32(ym))
    assert rel_err(got, want) < 2e-4


def test_deep_readout(lm_files):
    _torch()
    cfg = O.make_config(**dict(SMALL, post_merge_dims=[128], post_merge_activation="relu", maxout_pieces=1))
    cfg["post_merge_dims"] = [128, 64]
    base = O.init_params(dict(cfg, post_merge_dims=[128]), seed=31, scale=10.0)
    rng = np.random.RandomState(5)
    params = {}
    for k, v in base.items():
        if k.startswith(RO.PM + "/mlp/"):
            continue
        params[k] = v
        if k == RO.PM + "/bias.b":
            for j, (din, dout) in enumerate(((128, 64), (64, cfg["num_phonemes"]))):
                params[RO.linear_name(j) + ".b"] = rng.normal(0, 0.3, size=(dout,))
                params[RO.linear_name(j) + ".W"] = rng.normal(0, 1.5 / np.sqrt(din), size=(din, dout))
    x, xm, y, ym = O.synthetic_batch(cfg, B=3, T=30, seed=51)
    lm = lm_files(cfg["num_phonemes"])
    o = dict(DECODE_TLE, weight=0.5, no_transition_cost=20.0)
    rec = _rec(cfg, params, lm, o, "mse_gain", -5.0)
    got = rec.cost(x, xm, y, ym)
    p = _p64(params)
    a64, am64 = _attended(cfg, RO.shallow_params(cfg, params), x, xm)
    r = O.cost_matrix(cfg, RO.shallow_params(cfg, p), a64, am64, y, f32(ym), return_all=True)
    logits = RO.readout(cfg, p, r["states"], r["weighted_averages"])
    want = TLO.cost_of_logits(cfg, lm[2], o, dict(name="mse_gain", min_reward=-5.0), logits, y, f32(ym))
    assert rel_err(got, want) < 2e-4


def test_content_attention(lm_files):
    _torch()
    cfg, params, (x, xm, y, ym) = _setup(SMALL, seed=33, module=CO)
    lm = lm_files(cfg["num_phonemes"])
    o = dict(DECODE_TLE, weight=0.5, no_transition_cost=20.0)
    rec = _rec(cfg, params, lm, o, "mse_reward", -5.0)
    got = rec.cost(x, xm, y, ym)
    p = _p64(params)
    a64, am64 = O.encoder(cfg, p, f32(x), f32(xm))
    want = TLO.cost_matrix(cfg, p, lm[2], o, a64, am64, y, f32(ym), dict(name="mse_reward", min_reward=-5.0),
                           oracle=CO)
    assert rel_err(got, want) < 2e-4


@pytest.mark.parametrize("V", [5, 63, 128])
def test_vocabulary_widths(lm_files, V):
    _torch()
    cfg, params, (x, xm, y, ym) = _setup(dict(SMALL, num_phonemes=V), seed=35 + V)
    lm = lm_files(V)
    o = dict(DECODE_TLE, weight=0.5, no_transition_cost=20.0, normalize_tot_weights=True)
    rec = _rec(cfg, params, lm, o, "mse_gain", -1.0)
    a64, am64 = _attended(cfg, params, x, xm)
    want = TLO.cost_matrix(cfg, _p64(params), lm[2], o, a64, am64, y, f32(ym), dict(name="mse_gain"))
    assert rel_err(rec.cost(x, xm, y, ym), want) < 2e-4
    got = rec.generate(x, xm, n_steps=5, sample=False)
    outs, costs, _ = TLO.generate_greedy(cfg, _p64(params), lm[2], o, a64, am64, 5)
    np.testing.assert_array_equal(got["outputs"], outs)
    assert rel_err(got["costs"], costs) < 1e-4


def test_non_default_stream(lm_files):
    torch = _torch()
    cfg, params, (x, xm, y, ym) = _setup(SMALL, seed=37)
    lm = lm_files(cfg["num_phonemes"])
    o = dict(DECODE_TLE, weight=0.5, no_transition_cost=20.0)
    rec = _rec(cfg, params, lm, o, "mse_reward", -5.0)
    want = rec.cost(x, xm, y, ym)
    gen = rec.generate(x, xm, n_steps=5, sample=False)
    s = torch.cuda.Stream(device=rec.device)
    with torch.cuda.stream(s):
        np.testing.assert_array_equal(rec.cost(x, xm, y, ym), want)
        att, attm = rec.encode(x, xm)
        got = rec.cost_matrix(y, ym, att, attm)
        again = rec.generate(x, xm, n_steps=5, sample=False)
    s.synchronize()
    np.testing.assert_array_equal(got.cpu().numpy(), want)
    np.testing.assert_array_equal(again["outputs"], gen["outputs"])
    np.testing.assert_array_equal(again["costs"], gen["costs"])


def test_training_refusal_and_attach_order(lm_files):
    """The C entry points refuse a TLE handle with an LM before any device work; an LM attached before or after the
    criterion gives the same costs; pickling reloads both."""
    torch = _torch()
    cfg, params, (x, xm, y, ym) = _setup(SMALL, seed=39, B=2, T=24)
    lm = lm_files(cfg["num_phonemes"])
    o = dict(DECODE_TLE, weight=0.5, no_transition_cost=20.0)
    rec = _rec(cfg, params, lm, o, "mse_gain", -5.0)
    want = rec.cost(x, xm, y, ym)
    lib, h = package()._lib.load(), rec._require_ready()
    T, B, L = x.shape[0], x.shape[1], y.shape[0]
    n = sum(int(np.prod(s)) for s in rec.parameter_shapes().values())
    X = torch.as_tensor(x, device=rec.device)
    Y = torch.as_tensor(y, device=rec.device)
    grads = torch.zeros((4 * n,), dtype=torch.float32, device=rec.device)
    cost = torch.zeros((1,), dtype=torch.float32, device=rec.device)
    pred = torch.zeros((L + 10, B), dtype=torch.int64, device=rec.device)
    pmask = torch.zeros((L + 10, B), dtype=torch.float32, device=rec.device)
    lib.lvsr_launch_count(1)
    assert lib.lvsr_train_cost_and_grads(h, X.data_ptr(), None, Y.data_ptr(), None, T, B, L, 1.0, cost.data_ptr(),
                                         grads.data_ptr(), rec._stream()) != 0
    assert "language model" in lib.lvsr_last_error().decode()
    assert lib.lvsr_train_cost_and_grads_greedy(h, X.data_ptr(), None, Y.data_ptr(), T, B, L, 1.0, cost.data_ptr(),
                                                grads.data_ptr(), pred.data_ptr(), pmask.data_ptr(),
                                                rec._stream()) != 0
    assert "language model" in lib.lvsr_last_error().decode()
    assert lib.lvsr_launch_count(1) == 0
    torch.cuda.synchronize()
    assert float(grads.abs().max()) == 0.0 and float(cost[0]) == 0.0
    np.testing.assert_array_equal(rec.cost(x, xm, y, ym), want)       # the handle stays usable
    # criterion first, LM second (the recognizer attaches the LM first)
    other = make_recognizer(cfg, params, criterion=dict(name="mse_gain", min_reward=-5.0))
    other.cost(x, xm, y, ym)
    other.lm = package().recognizer._lm_config(dict(o, path=lm[0]))
    other.character_map = lm[1]
    other._lm_tables = package().lm.load(lm[0], lm[1], cfg["num_phonemes"])
    other._attach_lm(lib, other._require_ready())
    np.testing.assert_array_equal(other.cost(x, xm, y, ym), want)
    clone = pickle.loads(pickle.dumps(rec))
    assert clone.tle and clone.lm == rec.lm
    np.testing.assert_array_equal(clone.cost(x, xm, y, ym), want)


# ---- compat ----------------------------------------------------------------------------------------------------

def test_compat_search_with_decode_tle_overrides(tmp_path, capsys):
    _torch()
    import compat_helpers as CH
    if CH.COMPAT not in sys.path:
        sys.path.insert(0, CH.COMPAT)
    import lvsr.config as C
    import lvsr.main as M
    exp = CH.write_experiment(tmp_path)
    chars = list("abcdefghijk") + ["$"]
    S, start, arcs = LO.char_ngram(len(chars), seed=1, n_tri=8)
    fst_path = str(tmp_path / "LG_pushed_withsyms.fst")
    LO.to_file(fst_path, len(chars), S, start, arcs, seed=3)
    with open(fst_path, "rb") as f:                      # the data's characters as the FST's input symbols
        blob = f.read()
    for k in reversed(range(len(chars))):
        old, new = ("c%d" % k).encode(), chars[k].encode()
        blob = blob.replace(len(old).to_bytes(4, "little") + old, len(new).to_bytes(4, "little") + new)
    with open(fst_path, "wb") as f:
        f.write(blob)
    cfg = C.Configuration(exp["base"], None, [("net.criterion", "{name: mse_gain, min_reward: -5}"),
                                              ("monitoring.search.beam_size", "3"), ("net.lm.weight", "0.15"),
                                              ("net.lm.path", repr(fst_path))])
    assert cfg["net"]["lm"]["path"] == fst_path and cfg["net"]["criterion"]["name"] == "mse_gain"
    decoded = str(tmp_path / "decoded.txt")
    M.search(cfg, None, None, "valid", None, None, decoded, False, 1)
    out = capsys.readouterr().out
    for line in ("Groundtruth cost:", "Beam search cost:", "Recognized:", "Average CER:"):
        assert line in out, (line, out[-2000:])
    with open(decoded) as f:
        rows = f.read().splitlines()
    assert len(rows) == 3 and all(r.startswith("valid_") for r in rows), rows
    assert os.path.getsize(decoded) > 0
