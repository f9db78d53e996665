"""FST language model shallow fusion on the GPU against the float64 oracle (tests/lm_oracle.py): the LM state kernels
along random label walks, their error reports, the fused teacher-forced costs for every normalisation setting, the
fused beam search, pickling and the compat search entry point."""
import os
import pickle

import numpy as np
import pytest

import content_oracle as CO
import lm_oracle as LO
from helpers import O, PYRAMID, package

pytestmark = pytest.mark.gpu

V = PYRAMID["num_phonemes"]


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


@pytest.fixture(scope="module")
def lm_file(tmp_path_factory):
    S, start, arcs = LO.char_ngram(V, seed=7, n_tri=60, dup=6, dead=2)
    path = str(tmp_path_factory.mktemp("lm") / "lm.fst")
    cmap = LO.to_file(path, V, S, start, arcs, seed=2)
    return path, cmap, LO.from_tables(package().lm.load(path, cmap, V))


def _recognizer(cfg, params, lm=None, cmap=None):
    pkg = package()
    content = cfg.get("attention_type") == "content"
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": cfg["num_features"]}, input_num_chars={}, eos_label=cfg["eos_label"],
        num_phonemes=cfg["num_phonemes"], dim_dec=cfg["dim_dec"], dims_bidir=cfg["dims_bidir"],
        subsample=cfg["subsample"], conv_n=None if content else cfg["conv_n"],
        conv_num_filters=1 if content else cfg["conv_num_filters"], dim_matcher=cfg["dim_matcher"],
        post_merge_dims=cfg["post_merge_dims"], post_merge_activation=pkg.Maxout(cfg["maxout_pieces"]),
        dim_output_embedding=cfg["dim_feedback"], prior=None if content else cfg["prior"],
        attention_type="content" if content else "content_and_conv",
        max_decoded_length_scale=cfg["max_decoded_length_scale"], enc_transition=pkg.GatedRecurrent,
        dec_transition=pkg.GatedRecurrent, data_prepend_eos=False, lm=lm, character_map=cmap)
    rec.set_parameter_values(params)
    return rec


def _set(states, weights):
    return {int(s): float(w) for s, w in zip(states, weights) if s >= 0}


def _check_rows(st, sets, rows):
    gs, gw, ga = (st[k].cpu().numpy() for k in ("lm_states", "lm_weights", "lm_add"))
    for r, (want, row) in enumerate(zip(sets, rows)):
        got = _set(gs[r], gw[r])
        assert set(got) == set(want), (r, got, want)
        for s, w in want.items():
            assert abs(got[s] - w) <= 1e-9 * max(1.0, abs(w)), (r, s, got[s], w)
        assert np.allclose(ga[r], row, rtol=1e-5, atol=1e-5), (r, ga[r], row)


@pytest.mark.parametrize("ntc", [20.0, 1e12])
def test_lm_states_follow_the_oracle_along_random_walks(lm_file, ntc):
    _torch()
    path, cmap, fst = lm_file
    cfg = O.make_config(**PYRAMID)
    rec = _recognizer(cfg, O.init_params(cfg, seed=1), lm=dict(path=path, no_transition_cost=ntc), cmap=cmap)
    R, steps = 48, 25
    rng = np.random.RandomState(3)
    st = rec._lm_initial_states(R)
    s0, row0 = LO.initial(fst, V, ntc)
    sets, rows = [dict(s0) for _ in range(R)], [row0] * R
    _check_rows(st, sets, rows)
    dead = sizes = 0
    for _ in range(steps):
        # mostly symbols the LM knows, sometimes any symbol (hypotheses that leave the LM stay dead)
        y = np.array([rng.choice(np.flatnonzero(row < np.float32(ntc))) if (row < np.float32(ntc)).any() and rng.rand() < 0.9
                      else rng.randint(V) for row in rows], dtype=np.int64)
        st = rec._lm_next_states(st, y)
        nxt = [LO.next_state(fst, s, yy, V, ntc) for s, yy in zip(sets, y)]
        sets, rows = [n[0] for n in nxt], [n[1] for n in nxt]
        _check_rows(st, sets, rows)
        dead += sum(1 for s in sets if not s)
        sizes = max(sizes, max(len(s) for s in sets))
    print("dead rows over the walk:", dead, "largest set:", sizes)
    assert dead > 0 and sizes >= 3


def _error_fst(tmp_path):
    """a -> 1 -> a -> epsilon cycle; b -> 13 -> b -> nine states; c -> 14 (no arcs)."""
    a, b, c = 1, 2, 3
    arcs = [[] for _ in range(24)]
    arcs[0] = [(a, 1, 1.0), (b, 13, 1.0), (c, 14, 1.0)]
    arcs[1] = [(a, 2, 1.0)]
    arcs[2] = [(0, 3, 1.0)]
    arcs[3] = [(0, 2, 1.0)]
    arcs[13] = [(b, s, 1.0) for s in range(15, 24)]
    path = str(tmp_path / "bad.fst")
    return path, LO.to_file(path, V, 24, 0, arcs, seed=0)


def test_lm_errors_are_reported_and_the_handle_keeps_working(tmp_path):
    torch = _torch()
    path, cmap = _error_fst(tmp_path)
    cfg = O.make_config(**PYRAMID)
    rec = _recognizer(cfg, O.init_params(cfg, seed=1), lm=dict(path=path, no_transition_cost=20.0), cmap=cmap)
    init = rec._lm_initial_states(1)
    y = lambda v: torch.tensor([v], dtype=torch.int64)
    ok = rec._lm_next_states(init, y(2))
    assert _set(ok["lm_states"][0].cpu().numpy(), ok["lm_weights"][0].cpu().numpy()) == {14: 1.0}
    with pytest.raises(RuntimeError, match="epsilon cycle"):
        rec._lm_next_states(init, y(0))
    mid = rec._lm_next_states(init, y(1))
    with pytest.raises(RuntimeError, match="more than 7"):
        rec._lm_next_states(mid, y(1))
    again = rec._lm_next_states(init, y(2))
    assert torch.equal(again["lm_add"], ok["lm_add"]) and (again["lm_add"] == 20.0).all()
    # the search reports the error as well, and the handle searches afterwards
    rng = np.random.RandomState(0)
    x = rng.normal(size=(40, cfg["num_features"])).astype(np.float32)
    rec.init_beam_search(2)
    for _ in range(2):
        try:
            rec.beam_search({"recordings": x})
        except (RuntimeError, package().CandidateNotFoundError):
            pass
    assert torch.equal(rec._lm_next_states(init, y(2))["lm_add"], ok["lm_add"])


FLAGS = [dict(normalize_am_weights=a, normalize_lm_weights=l, normalize_tot_weights=t)
         for a in (True, False) for l in (True, False) for t in (True, False)]


@pytest.mark.parametrize("stepwise", [False, True], ids=["persistent", "stepwise"])
@pytest.mark.parametrize("attention", ["content_and_conv", "content"])
def test_fused_cost_matrix_equals_oracle(lm_file, attention, stepwise, monkeypatch):
    torch = _torch()
    path, cmap, fst = lm_file
    if stepwise:
        monkeypatch.setenv("LVSR_NO_DEC_SCAN", "1")
    M = CO if attention == "content" else O
    cfg = M.make_config(**PYRAMID)
    params = M.init_params(cfg, seed=4, scale=10.0)
    x, m, labels, lmask = O.synthetic_batch(cfg, B=3, T=40, seed=5)
    att, attm = O.encoder(cfg, params, x, m)
    r = M.cost_matrix(cfg, params, att, attm, labels, lmask, return_all=True)
    logits = O.readout(cfg, params, r["states"], r["weighted_averages"])
    rec = _recognizer(cfg, params, lm=dict(path=path, no_transition_cost=20.0), cmap=cmap)
    lib, h = package()._lib.load(), rec._require_ready()
    gatt, gattm = rec.encode(x, m)
    n = 0
    for ntc in (20.0, 1e12):
        add = LO.lm_path(fst, labels, lmask, V, ntc)
        for flags in FLAGS:
            for am_beta in (1.0, 0.7):
                for weight in (0.0, 0.5):
                    if ntc > 100 and flags["normalize_tot_weights"]:
                        continue           # a log_softmax over a row of ~1e12 entries is float32 noise in the reference too
                    o = dict(flags, am_beta=am_beta, weight=weight, no_transition_cost=ntc)
                    rec.lm.update(o)
                    rec._attach_lm(lib, h)
                    got = rec.cost_matrix(labels, lmask, gatt, gattm).cpu().numpy().astype(np.float64)
                    want = np.take_along_axis(LO.fused_costs(logits, add, o), labels[..., None], axis=-1)[..., 0] * lmask
                    assert np.allclose(got, want, rtol=1e-4, atol=1e-4), (o, np.abs(got - want).max())
                    n += 1
    print("settings compared:", n)
    # analyze / cost go through the same fused path
    rec.lm.update(dict(FLAGS[0], am_beta=1.0, weight=0.5, no_transition_cost=20.0))
    rec._attach_lm(lib, h)
    want = LO.cost_matrix(cfg, params, fst, rec.lm, att, attm, labels, lmask, oracle=M)
    assert np.allclose(rec.cost(x, m, labels, lmask), want, rtol=1e-4, atol=1e-4)


def _peaky(cfg, seed, gain=10.0, eos_bias=1.0):
    params = O.init_params(cfg, seed=seed, scale=10.0)
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.W"] *= gain
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.b"][cfg["eos_label"]] = eos_bias
    return params


@pytest.mark.parametrize("prior", [None, dict(type="window_around_median", before=6, after=8)],
                         ids=["default", "median"])
@pytest.mark.parametrize("beam_size,stop_on,char_discount", [(1, "patience", 0), (5, "patience", 0.0),
                                                             (10, "optimistic_future_cost", 0.1)])
def test_fused_search_many_equals_oracle(lm_file, prior, beam_size, stop_on, char_discount):
    _torch()
    path, cmap, fst = lm_file
    cfg = O.make_config(prior=prior, max_decoded_length_scale=3.0, **PYRAMID)
    params = _peaky(cfg, 11)
    o = dict(LO_DEFAULTS, weight=0.5, no_transition_cost=20.0)
    rec = _recognizer(cfg, params, lm=dict(o, path=path), cmap=cmap)
    rng = np.random.RandomState(5)
    utts = [rng.normal(size=(T, cfg["num_features"])) for T in (64, 37, 52, 45)]
    rec.init_beam_search(beam_size)
    got = rec._beam_search.search_many([u.astype(np.float32) for u in utts], cfg["eos_label"],
                                       [int(u.shape[0] / 3.0) for u in utts], stop_on=stop_on,
                                       char_discount=char_discount, raise_on_failure=False)
    comp = LO.computers(cfg, params, fst, o)
    n_found = n_hyp = 0
    for u, g in zip(utts, got):
        try:
            want = O.beam_search(cfg, params, u, beam_size, stop_on=stop_on, char_discount=char_discount,
                                 computers=comp)
        except O.CandidateNotFoundError:
            assert g is None
            continue
        assert g is not None
        n_found += 1
        n_hyp += len(want[0])
        assert g[0] == want[0]
        assert np.allclose(g[1], want[1], rtol=1e-3, atol=5e-3)
    print("utterances with a result:", n_found, "finished hypotheses compared:", n_hyp)
    if beam_size >= 5:
        assert n_found >= 1 and n_hyp >= 3


LO_DEFAULTS = dict(normalize_am_weights=True, normalize_lm_weights=False, normalize_tot_weights=False, am_beta=1.0)


def test_weight_zero_searches_like_no_lm_and_launches_do_not_grow_with_utterances(lm_file):
    _torch()
    path, cmap, fst = lm_file
    cfg = O.make_config(max_decoded_length_scale=3.0, **PYRAMID)
    params = _peaky(cfg, 11)
    rng = np.random.RandomState(6)
    utts = [rng.normal(size=(T, cfg["num_features"])).astype(np.float32) for T in (60, 41, 52, 48, 33, 57)]
    maxl = [int(u.shape[0] / 3.0) for u in utts]
    plain, zero = _recognizer(cfg, params), _recognizer(cfg, params, lm=dict(path=path, weight=0.0), cmap=cmap)
    for rec in (plain, zero):
        rec.init_beam_search(5)
    a = plain._beam_search.search_many(utts, cfg["eos_label"], maxl, raise_on_failure=False)
    b = zero._beam_search.search_many(utts, cfg["eos_label"], maxl, raise_on_failure=False)
    assert [None if r is None else r[0] for r in a] == [None if r is None else r[0] for r in b]
    assert any(r is not None for r in a)
    lib = package()._lib.load()
    weighted = _recognizer(cfg, params, lm=dict(path=path, weight=0.5, no_transition_cost=20.0), cmap=cmap)
    weighted.init_beam_search(4)
    lib.lvsr_launch_count(1)
    weighted._beam_search.search_many(utts[:1], cfg["eos_label"], [12], raise_on_failure=False)
    one = lib.lvsr_launch_count(1)
    weighted._beam_search.search_many(utts * 2, cfg["eos_label"], [12] * 12, raise_on_failure=False)
    many = lib.lvsr_launch_count(1)
    print("launches: 1 utterance", one, "12 utterances", many)
    assert many <= 1.5 * one


def test_pickle_round_trip_reloads_the_lm(lm_file):
    _torch()
    path, cmap, fst = lm_file
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=4, scale=10.0)
    x, m, labels, lmask = O.synthetic_batch(cfg, B=2, T=32, seed=9)
    rec = _recognizer(cfg, params, lm=dict(path=path, weight=0.5, no_transition_cost=20.0), cmap=cmap)
    before = rec.cost(x, m, labels, lmask)
    back = pickle.loads(pickle.dumps(rec))
    assert np.array_equal(back.cost(x, m, labels, lmask), before)
    plain = _recognizer(cfg, params)
    assert not np.allclose(plain.cost(x, m, labels, lmask), before)


def test_compat_search_with_an_lm_path(tmp_path, capsys):
    _torch()
    import sys
    import compat_helpers as CH
    if CH.COMPAT not in sys.path:
        sys.path.insert(0, CH.COMPAT)
    import lvsr.config as C
    import lvsr.main as M
    exp = CH.write_experiment(tmp_path)
    chars = list("abcdefghijk") + ["$"]
    S, start, arcs = LO.char_ngram(len(chars), seed=1, n_tri=8)
    fst_path = str(tmp_path / "lm.fst")
    cmap = LO.to_file(fst_path, len(chars), S, start, arcs, seed=3)
    # the same FST with the data's characters as its input symbols
    with open(fst_path, "rb") as f:
        blob = f.read()
    for k in reversed(range(len(chars))):
        old, new = ("c%d" % k).encode(), chars[k].encode()
        blob = blob.replace(len(old).to_bytes(4, "little") + old, len(new).to_bytes(4, "little") + new)
    with open(fst_path, "wb") as f:
        f.write(blob)
    vocab = str(tmp_path / "words.txt")
    with open(vocab, "w") as f:
        f.write("<UNK> 0\n")
    cfg = C.Configuration(exp["base"], None, [("monitoring.search.beam_size", "2"), ("net.lm.path", repr(fst_path)),
                                              ("net.lm.weight", "0.5"), ("net.lm.no_transition_cost", "20"),
                                              ("vocabulary", repr(vocab))])
    assert cfg["net"]["lm"]["path"] == fst_path
    M.search(cfg, None, None, "valid", None, None, None, False, 1)
    out = capsys.readouterr().out
    assert "Average CER:" in out and "Average WER:" in out
