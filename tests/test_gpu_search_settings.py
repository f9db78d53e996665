"""Beam search at the settings the reference decodes with: beam 200 (exp/wsj/README.md, decode.sh), ignore_first_eol
(SpeechRecognizer.beam_search passes data_prepend_eos, True by default), round_to_inf 4.5 (the TIMIT / WSJ reward
recipes), char_discount 0.1 / 1.0, a validate_solution_function and LM fusion at decode.sh's weights.

At beam 200 the k-th and (k+1)-th of thousands of candidates are routinely within float32 rounding of each other, so
token lists cannot be compared with the float64 oracle's.  Two kinds of check instead:

  * An exact replay.  O.beam_search (the line-for-line BeamSearch.search) runs over the recognizer's own device state
    functions (_initial_states, _logprobs, _next_states) on the contexts of the same batched encode / preprocess that
    search_many makes, with every row reading its own utterance (row_utt), float32 costs, and its selection replaced
    by segment_topk_kernel's documented rule: a stable sort on (cost, flat index).  With LVSR_ATT_CS=1 a glimpse is
    computed by one CTA whatever the row count, and dense_kernel and readout_kernel compute each row on its own, so
    lvsr_beam_search_many must give the replay's token histories, float32 cost histories and `done` order bit for
    bit.  The utterances have equal lengths: lvsr_logprobs clips the expanding window at T', not at the utterance's
    length.  Most cases give two symbols the same readout column, so exact ties at the k boundary are met all the
    time and settle by the flat index; the replay counts them.
  * Float64 anchors that do not depend on ties: every returned hypothesis' cumulative costs against the teacher-forced
    O.cost_matrix of its own tokens (priors under which a row's glimpse does not depend on the rest of the beam, and
    LM fusion at decode.sh's settings), and searches of 3 steps at k = 200 compared with O.beam_search wherever every
    k boundary has a float64 gap of at least 1e-3.  The oracle is given the GPU's encoder output and the parameters
    rounded to float32, so the errors measured are the decoder's and the search's.

Every case asserts from the replay's counters (O.beam_search's `stats`) that its setting decided something: a
stopping criterion ended a search before max_length, round_to_inf removed eol hypotheses, eol was kept in the beam at
step 0, the validator rejected hypotheses.

Measured on an H100 80GB HBM3 (700 W power limit): every replay agreed bit for bit, with 397 to 878 exact ties at
or inside the k boundary per prior of the beam-200 matrix; worst cumulative cost errors 2.2e-6 (default prior),
8.9e-7 (expanding), 2.1e-6 (content), 1.4e-6 with the LM and 5.7e-7 over the 3-step searches (all 12 utterances
qualified), bound 1e-5.  The file runs in about 25 s.
"""
import time
from collections import OrderedDict

import numpy as np
import pytest

import bench
import content_oracle as CO
import lm_oracle as LO
import stack_oracle as SO
from helpers import O, PYRAMID, elementwise_err, f32, make_recognizer, package

pytestmark = pytest.mark.gpu

RO = "/recognizer/generator/readout/post_merge/mlp/linear_0"
TIE = (3, 4)                   # symbol 4 reads out exactly like symbol 3
SEARCH_COST_TOL = 1e-5         # cumulative costs of the returned hypotheses (test_gpu_widths.py's search_costs)


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


@pytest.fixture(autouse=True)
def _one_cta_per_glimpse(monkeypatch):
    monkeypatch.setenv("LVSR_ATT_CS", "1")


def _peaky(cfg, seed, M=O, gain=10.0, eos_bias=1.0, tie=True):
    """Parameters whose readout is sharp enough that hypotheses of many lengths finish (test_gpu_search.py); with
    `tie`, symbols TIE have one readout column, so their costs are equal in every row."""
    params = M.init_params(cfg, seed=seed, scale=10.0)
    params[RO + ".W"] *= gain
    params[RO + ".b"][cfg["eos_label"]] = eos_bias
    if tie:
        params[RO + ".W"][:, TIE[1]] = params[RO + ".W"][:, TIE[0]]
        params[RO + ".b"][TIE[1]] = params[RO + ".b"][TIE[0]]
    return params


def _utts(F, lens, seed):
    rng = np.random.RandomState(seed)
    return [rng.normal(size=(T, F)).astype(np.float32) for T in lens]


def _contexts(rec, utts):
    """The contexts BeamSearch.search_many builds: one encode of the right-padded utterances, then preprocess."""
    lens = [u.shape[0] for u in utts]
    x = np.zeros((max(lens), len(utts), utts[0].shape[1]), dtype=np.float32)
    for j, u in enumerate(utts):
        x[:lens[j], j] = u
    mask = None if min(lens) == max(lens) else (np.arange(max(lens))[:, None] < np.asarray(lens)[None, :]).astype(np.float32)
    att, attm = rec.encode(x, mask)
    return dict(attended=att, attended_mask=attm, preprocessed=rec.preprocess(att))


def _device_computers(rec, ctx, u):
    """O.beam_search's state functions on the device: utterance u of the batched contexts for every row."""
    torch = _torch()
    Tp = ctx["attended"].shape[0]

    def host(st):
        return OrderedDict((k, v.cpu().numpy()) for k, v in st.items())

    def dev(st):
        return {k: torch.as_tensor(np.ascontiguousarray(st[k]), device=rec.device) for k in ("states", "weights", "step")}

    def rows(st):
        return dict(ctx, row_utt=torch.full((st["states"].shape[0],), u, dtype=torch.int32, device=rec.device))

    dummy = np.zeros((1, 1, 1), np.float32)          # only its dtype is used: the replay's costs are float32
    return dict(context=lambda x: (dummy, dummy[:, :, 0]),
                initial=lambda att: host(rec._initial_states(Tp, 1)),
                logprobs=lambda att, m, st: rec._logprobs(rows(st), dev(st)).cpu().numpy(),
                next=lambda att, m, st, y: host(rec._next_states(rows(st), dev(st), y)))


class Selection:
    """BeamSearch._smallest with segment_topk_kernel's order: a stable sort on (cost, flat index).  Counts the exact
    ties among the selected candidates and the first one left out, and the widest candidate table."""

    def __init__(self):
        self.ties = 0
        self.rows = 0

    def __call__(self, matrix, k):
        flat = matrix.reshape(-1)
        order = np.argsort(flat, kind="stable")
        keep = order[:min(k, flat.shape[0])]
        head = flat[order[:k + 1]]
        self.ties += int(np.count_nonzero(head[1:] == head[:-1]))
        self.rows = max(self.rows, matrix.shape[0])
        return np.unravel_index(keep, matrix.shape), flat[keep]


def _replay(monkeypatch, sel, rec, ctx, u, x, k, max_length, **kw):
    """O.beam_search over the device state functions -> (ranked done [(tokens, float32 costs)], stats)."""
    monkeypatch.setattr(O, "smallest", sel)
    stats = {}
    try:
        done = O.beam_search(None, None, x, k, eol_symbol=rec.eos_label, max_length=max_length,
                             computers=_device_computers(rec, ctx, u), as_arrays=True, stats=stats, **kw)
    except O.CandidateNotFoundError:
        done = []
    return done, stats


def _histories(rec, result):
    """An as_arrays result of search_many back to the ranked `done` list: [(tokens with the initial symbol, cumulative
    float32 costs from 0)].  The float64 differences of float32 costs are exact, and so are their partial sums."""
    if result is None:
        return []
    outputs, masks, steps = result
    out = []
    for j in range(outputs.shape[1]):
        n = int(masks[:, j].sum())
        tok = np.concatenate([[rec.net["num_phonemes"]], outputs[:n, j]]).astype(np.int64)
        cost = np.concatenate([[0.0], np.cumsum(steps[:n, j])])
        assert np.array_equal(cost.astype(np.float32).astype(np.float64), cost)
        out.append((tok, cost.astype(np.float32)))
    return out


def _assert_same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for j, ((gt, gc), (wt, wc)) in enumerate(zip(got, want)):
        assert np.array_equal(gt, wt), (what, j, gt, wt)
        assert wc.dtype == np.float32 and np.array_equal(gc, wc), (what, j, gc, wc)


def _search_and_replay(monkeypatch, rec, utts, k, max_lengths, sel, replay=None, **kw):
    """search_many over all utterances, each of `replay` (default: all) replayed; -> (results, [stats])."""
    rec.init_beam_search(k)
    got = rec._beam_search.search_many(utts, rec.eos_label, max_lengths, as_arrays=True, raise_on_failure=False, **kw)
    ctx = _contexts(rec, utts)
    stats = []
    for u in (range(len(utts)) if replay is None else replay):
        want, st = _replay(monkeypatch, sel, rec, ctx, u, utts[u], k, max_lengths[u], **kw)
        _assert_same(_histories(rec, got[u]), want, (u, kw))
        stats.append(st)
    return got, stats


# ---- 1. beam 200, every prior and content attention, both stopping criteria x char_discount ---------------------

MEDIAN = dict(type="window_around_median", before=6, after=8)
MEAN = dict(type="window_around_mean", before=7, after=7)
EXPANDING = dict(type="expanding", initial_begin=0, initial_end=6, min_speed=0.8, max_speed=2.5)
PRIORS = dict(default=None, expanding=EXPANDING, median=MEDIAN, mean=MEAN, content=None)
SETTINGS = [(stop_on, cd) for stop_on in ("patience", "optimistic_future_cost") for cd in (0.0, 0.1, 1.0)]
SCALE = 1.5                    # 64 frames -> max_length 42: patience (30 steps) can end a search before it


def _config(prior, M=O, **kw):
    return M.make_config(prior=prior, max_decoded_length_scale=SCALE, **dict(PYRAMID, **kw))


@pytest.mark.parametrize("prior", list(PRIORS))
def test_beam200_replays_exactly(prior, monkeypatch):
    """Every stopping criterion ends some search before max_length (the optimistic one once 200 hypotheses have
    finished, which its bound rarely allows at char_discount 1.0), and the char discount reorders some ranking."""
    _torch()
    M = CO if prior == "content" else O
    cfg = _config(PRIORS[prior], M)
    rec = make_recognizer(cfg, _peaky(cfg, 11, M, eos_bias=2.0))
    utts = _utts(cfg["num_features"], (64,) * 5, seed=5)
    sel, t0 = Selection(), time.time()
    fired, orders = {}, {}
    for stop_on, cd in SETTINGS:
        got, stats = _search_and_replay(monkeypatch, rec, utts, 200, [int(64 / SCALE)] * len(utts), sel,
                                        stop_on=stop_on, char_discount=cd)
        stopped = [s["stop"] for s in stats]
        print(prior, stop_on, cd, "stops", stopped, "finished", [s["finished"] for s in stats])
        fired[stop_on, cd] = sum(1 for s in stopped if s is not None)
        orders[stop_on, cd] = [None if r is None else r[0].T.tolist() for r in got]
        assert sum(s["finished"] for s in stats) >= 10
    print(prior, "exact ties at or inside the k boundary: %d, widest table %d rows, %.1f s" % (sel.ties, sel.rows, time.time() - t0))
    assert sel.ties > 0 and sel.rows == 200
    assert all(fired["patience", cd] for cd in (0.0, 0.1, 1.0)), fired
    assert fired["optimistic_future_cost", 0.0] or fired["optimistic_future_cost", 0.1], fired
    assert orders["patience", 0.0] != orders["patience", 1.0]


# ---- ignore_first_eol, round_to_inf, validator, stacked decoder ----------------------------------------------------

@pytest.mark.parametrize("k,eos_bias", [(200, 1.0), (5, 5.0)])
def test_ignore_first_eol_through_beam_search(k, eos_bias, monkeypatch):
    """data_prepend_eos=True: an eol chosen at step 0 is finished and stays in the beam (search.cu's ignore_first_eol
    branch).  At k = 200 > V eol is always chosen at step 0; at k = 5 the eos bias puts it in the first top 5."""
    _torch()
    cfg = _config(None)
    rec = make_recognizer(cfg, _peaky(cfg, 11, eos_bias=eos_bias))
    rec.data_prepend_eos = True
    rec.init_beam_search(k)
    eol, kept, continued = cfg["eos_label"], 0, 0
    sel = Selection()
    for x in _utts(cfg["num_features"], (64, 64, 64), seed=5):
        got = _histories(rec, rec.beam_search({"recordings": x}, as_arrays=True))
        want, st = _replay(monkeypatch, sel, rec, _contexts(rec, [x]), 0, x, k, int(64 / SCALE), ignore_first_eol=True)
        _assert_same(got, want, ("ignore_first_eol", k))
        kept += st["eol_kept_first"]
        continued += sum(1 for t, _ in got if t[1] == eol and len(t) > 2)      # a finished child of a step-0 eol
    print("k", k, "step-0 eol kept:", kept, "finished hypotheses continuing one:", continued, "ties:", sel.ties)
    assert kept == 3 and continued > 0


def test_round_to_inf_with_patience(monkeypatch):
    """round_to_inf 4.5 with patience (exp/timit/configs/iclr_reward.yaml): an eol whose step costs 4.5 or more neither
    finishes nor stays in the beam."""
    _torch()
    cfg = _config(MEDIAN)
    rec = make_recognizer(cfg, _peaky(cfg, 11))
    utts = _utts(cfg["num_features"], (64, 64, 64), seed=5)
    sel = Selection()
    _, stats = _search_and_replay(monkeypatch, rec, utts, 200, [int(64 / SCALE)] * 3, sel, round_to_inf=4.5)
    removed, finished = sum(s["eol_removed"] for s in stats), sum(s["finished"] for s in stats)
    print("eol removed by round_to_inf:", removed, "finished:", finished, "ties:", sel.ties)
    assert removed > 0 and finished > 0


def test_validator_at_beam200(monkeypatch):
    """A validate_solution_function that keeps the hypotheses of even length (about half of them)."""
    _torch()
    cfg = _config(MEAN)
    rec = make_recognizer(cfg, _peaky(cfg, 11))
    utts = _utts(cfg["num_features"], (64, 64, 64), seed=8)
    sel = Selection()
    _, stats = _search_and_replay(monkeypatch, rec, utts, 200, [int(64 / SCALE)] * 3, sel,
                                  validate_solution_function=lambda inputs, seq: len(seq) % 2 == 0)
    rejected, finished = sum(s["rejected"] for s in stats), sum(s["finished"] for s in stats)
    print("validator kept", finished, "rejected", rejected, "ties:", sel.ties)
    assert finished > 0 and rejected > 0


def test_stacked_decoder_at_beam200(monkeypatch):
    _torch()
    cfg = SO.make_config(max_decoded_length_scale=SCALE, **PYRAMID)
    rec = make_recognizer(cfg, _peaky(cfg, 11, SO))
    utts = _utts(cfg["num_features"], (64, 64), seed=5)
    sel = Selection()
    _, stats = _search_and_replay(monkeypatch, rec, utts, 200, [int(64 / SCALE)] * 2, sel)
    print("stacked: stops", [s["stop"] for s in stats], "finished", [s["finished"] for s in stats], "ties", sel.ties)
    assert "patience" in [s["stop"] for s in stats] and sel.ties > 0


# ---- selection limits -----------------------------------------------------------------------------------------------

def test_selection_at_its_shared_memory_limits(monkeypatch):
    """V = 128: k = 200 takes 100 KB of opt-in shared memory, k = 400 exactly the 200 KB the kernel accepts; k = 401
    is refused with the kernel's message and the handle then searches as before.  At step 0 only V = 128 < k
    candidates exist."""
    _torch()
    cfg = O.make_config(max_decoded_length_scale=3.0, **dict(PYRAMID, num_phonemes=128))
    rec = make_recognizer(cfg, _peaky(cfg, 11))
    utts = _utts(cfg["num_features"], (64, 64), seed=5)
    maxl = [int(64 / 3.0)] * 2
    first = {}
    for k in (200, 400):
        sel = Selection()
        first[k], stats = _search_and_replay(monkeypatch, rec, utts, k, maxl, sel)
        print("V 128 k", k, "finished", [s["finished"] for s in stats], "ties", sel.ties, "rows", sel.rows)
        assert sel.rows == k and sum(s["finished"] for s in stats) > 0
    rec.init_beam_search(401)
    with pytest.raises(RuntimeError, match="beam_size 401 x 128 symbols does not fit the selection kernel"):
        rec._beam_search.search_many(utts, rec.eos_label, maxl, as_arrays=True, raise_on_failure=False)
    rec.init_beam_search(400)
    again = rec._beam_search.search_many(utts, rec.eos_label, maxl, as_arrays=True, raise_on_failure=False)
    for a, b in zip(first[400], again):
        _assert_same(_histories(rec, b), _histories(rec, a), "after the refusal")


# ---- configs[2]'s shape at beam 200 -------------------------------------------------------------------------------

def test_bench_search_shape_at_beam200(monkeypatch):
    """bench.py's configs[2] network and weights, 32 utterances x 800 frames in one search_many: 6400 rows per step
    while every beam is full.  A subset of the utterances is replayed."""
    _torch()
    cfg = O.make_config(max_decoded_length_scale=8.0, **bench.NET)
    rec = make_recognizer(cfg)
    rec.set_parameter_values(bench.search_values(rec.parameter_shapes()))
    utts = _utts(40, [800] * 32, seed=99)
    sel, t0 = Selection(), time.time()
    got, stats = _search_and_replay(monkeypatch, rec, utts, 200, [100] * 32, sel, replay=(0, 13, 31))
    print("configs[2] at beam 200: decoded %d of 32, replayed stops %s, ties %d, %.1f s" % (
        sum(r is not None for r in got), [s["stop"] for s in stats], sel.ties, time.time() - t0))
    assert sel.rows == 200 and all(s["finished"] > 0 for s in stats)


# ---- 3. float64 anchors -------------------------------------------------------------------------------------------

def _anchor(rec, cfg, params, utts, got, cost_matrix):
    """Worst elementwise_err of the returned hypotheses' cumulative costs against cost_matrix(attended, labels, mask) of
    their own tokens, one batched call per utterance on its own GPU encoding."""
    worst, n = 0.0, 0
    for x, res in zip(utts, got):
        hyps = _histories(rec, res)
        if not hyps:
            continue
        att, attm = rec.encode(x[:, None, :])
        H, L = len(hyps), max(len(t) for t, _ in hyps) - 1
        labels = np.zeros((L, H), np.int64)
        mask = np.zeros((L, H))
        for j, (t, _) in enumerate(hyps):
            labels[:len(t) - 1, j] = t[1:]
            mask[:len(t) - 1, j] = 1
        a64 = np.repeat(att.double().cpu().numpy(), H, axis=1)
        m64 = np.repeat(attm.double().cpu().numpy(), H, axis=1)
        want = np.cumsum(cost_matrix(a64, m64, labels, mask), axis=0)
        for j, (t, c) in enumerate(hyps):
            worst = max(worst, elementwise_err(c[1:], want[:len(t) - 1, j]))
        n += H
    return worst, n


@pytest.mark.parametrize("prior", ["default", "expanding", "content"])
def test_hypothesis_costs_equal_teacher_forced_oracle(prior):
    """(a) Ragged lengths at beam 200: every returned hypothesis' cumulative costs equal O.cost_matrix of its tokens."""
    _torch()
    M = CO if prior == "content" else O
    cfg = _config(PRIORS[prior], M)
    params = _peaky(cfg, 11, M)
    rec = make_recognizer(cfg, params)
    utts = _utts(cfg["num_features"], (64, 41, 55, 37), seed=6)
    rec.init_beam_search(200)
    got = rec._beam_search.search_many(utts, cfg["eos_label"], [int(u.shape[0] / SCALE) for u in utts],
                                       as_arrays=True, raise_on_failure=False, char_discount=0.1)
    p32 = {k: f32(v) for k, v in params.items()}
    worst, n = _anchor(rec, cfg, params, utts, got, lambda a, m, y, ym: M.cost_matrix(cfg, p32, a, m, y, ym))
    print(prior, "hypotheses", n, "worst cumulative cost error %.2e" % worst)
    assert n >= 20 and worst <= SEARCH_COST_TOL


@pytest.fixture(scope="module")
def lm_file(tmp_path_factory):
    """test_gpu_lm.py's trigram FST."""
    V = PYRAMID["num_phonemes"]
    S, start, arcs = LO.char_ngram(V, seed=7, n_tri=60, dup=6, dead=2)
    path = str(tmp_path_factory.mktemp("lm") / "lm.fst")
    cmap = LO.to_file(path, V, S, start, arcs, seed=2)
    return path, cmap, LO.from_tables(package().lm.load(path, cmap, V))


def test_lm_fused_hypothesis_costs_at_decode_settings(lm_file):
    """(b) exp/wsj/decode.sh with an LM: weight 0.5, no_transition_cost 20, char_discount 1.0, beam 200."""
    _torch()
    path, cmap, fst = lm_file
    cfg = _config(None)
    params = _peaky(cfg, 11)
    o = dict(normalize_am_weights=True, normalize_lm_weights=False, normalize_tot_weights=False, am_beta=1.0,
             weight=0.5, no_transition_cost=20.0)
    rec = make_recognizer(cfg, params, lm=dict(o, path=path), character_map=cmap)
    utts = _utts(cfg["num_features"], (64, 41, 55, 37), seed=6)
    rec.init_beam_search(200)
    got = rec._beam_search.search_many(utts, cfg["eos_label"], [int(u.shape[0] / SCALE) for u in utts],
                                       as_arrays=True, raise_on_failure=False, char_discount=1.0)
    p32 = {k: f32(v) for k, v in params.items()}
    worst, n = _anchor(rec, cfg, params, utts, got, lambda a, m, y, ym: LO.cost_matrix(cfg, p32, fst, o, a, m, y, ym))
    print("LM fused: hypotheses", n, "worst cumulative cost error %.2e" % worst)
    assert n >= 20 and worst <= SEARCH_COST_TOL


def test_three_steps_against_float64_oracle(monkeypatch):
    """(c) max_length 3 at k = 200, V = 32: the selections run over 32, 1 024 and up to 6 400 candidates.  An utterance
    is compared when every k boundary the float64 oracle meets has a gap of at least 1e-3; most must qualify."""
    _torch()
    cfg = _config(None)
    params = _peaky(cfg, 11, tie=False)          # the float64 oracle would meet the exact ties too
    rec = make_recognizer(cfg, params)
    utts = _utts(cfg["num_features"], [64, 48, 57, 40, 64, 52, 44, 61, 36, 64, 50, 45], seed=12)
    rec.init_beam_search(200)
    got = rec._beam_search.search_many(utts, cfg["eos_label"], [3] * len(utts), raise_on_failure=False)
    p32 = {k: f32(v) for k, v in params.items()}
    compared, worst, gaps = 0, 0.0, []

    def smallest(matrix, k):
        flat = np.sort(matrix.reshape(-1))
        if flat.shape[0] > k:
            gaps.append(flat[k] - flat[k - 1])
        return O_smallest(matrix, k)

    O_smallest = O.smallest
    monkeypatch.setattr(O, "smallest", smallest)
    for x, g in zip(utts, got):
        att, attm = rec.encode(x[:, None, :])
        ctx = (att.double().cpu().numpy(), attm.double().cpu().numpy())
        del gaps[:]
        want = O.beam_search(cfg, p32, x, 200, max_length=3, computers=dict(context=lambda r: ctx))
        assert len(gaps) == 2
        if min(gaps) < 1e-3:
            continue
        compared += 1
        assert g is not None and sorted(map(tuple, g[0])) == sorted(map(tuple, want[0]))
        rank = {tuple(t): c for t, c in zip(*want)}
        worst = max(worst, elementwise_err(g[1], [rank[tuple(t)] for t in g[0]]))
    print("compared %d of %d utterances, worst total cost error %.2e" % (compared, len(utts), worst))
    assert compared > len(utts) // 2 and worst <= SEARCH_COST_TOL
