"""The FST language model's kernels (csrc/lm.cu) and the fused readout against the float64 oracle of
tests/lm_oracle.py, at every vocabulary width, set size and closure they accept, on the benchmark's million-arc 4-gram
and at the benchmark's search shape.  The FSTs come from tests/lm_fixtures.py, generated from seeds; the CPU file
tests/test_lm_matrix_cpu.py shows that each one reaches what the case below claims.

  1. V in {2, 31, 33, 63, 64, 65, 127, 128}: LM state walks at R in {1, 3, 5, 4097}, and cost_matrix with the LM for
     every normalisation flag (both decoders at V = 63, content attention at V = 65).  V above 128 is refused when
     the handle is created.
  2. Sets of exactly 1 to 7 states, 8 refused; a cost-row candidate whose epsilon closure holds 32 states, and 33
     refused both as a candidate and as the taken transition.  After every refusal the handle repeats its results
     bit for bit.
  3. Closures whose discovery order is not a topological order (diamonds, parallel epsilon arcs, arcs back into the
     transition's set, chains 6 deep), mixed-sign weights, `standard` and `log` files.
  4. Walks of 320 symbols on the 4-gram and a weight-pushed (mixed-sign) variant: set weights in the hundreds.
  5. Teacher forcing with masks zero in the middle of rows, a row masked entirely, B = 64 x L = 300 and L = 1.
  6. The 4-gram with a start state of more than 1,000 arcs in runs of equal labels: 6,400 independent walks of 50
     steps, every row's set compared and the cost rows of a seeded sample of 256 rows per step.
  7. The fused search at bench.py's configs[2] shape (bench.NET, 32 utterances x 800 frames) at exp/wsj/decode.sh's
     fusion settings: beam 10 against O.beam_search, beam 200 against the teacher-forced oracle.

Bounds (those of test_gpu_lm.py): set weights 1e-9 relative (floor 1), cost rows rtol = atol = 1e-5, fused costs
1e-4, cumulative search costs 1e-5.  The walks of case 1 follow 32 distinct symbol sequences (row r the sequence
r mod 32) so that the oracle, memoised by frozen set, computes each set once; every row is compared.

The file ran in 170 s on an H100 80GB HBM3 (700 W power limit), almost all of it in the Python oracle: 57 s in case 7
(the beam-10 oracle searches and the beam-200 teacher-forced anchors), 46 s in case 6, 16 s in case 5 (64 x 300 rows)
and 16 s in the two long walks of case 4.
"""
import time

import numpy as np
import pytest

import bench
import content_oracle as CO
import lm_fixtures as F
import lm_oracle as LO
from helpers import O, PYRAMID, elementwise_err, f32, make_recognizer, package
from test_gpu_search_settings import _anchor

pytestmark = pytest.mark.gpu

NTC = 20.0
WIDTHS = [2, 31, 33, 63, 64, 65, 127, 128]
SET_TOL, ROW_TOL, FUSED_TOL, SEARCH_COST_TOL = 1e-9, 1e-5, 1e-4, 1e-5
DECODE = dict(normalize_am_weights=True, normalize_lm_weights=False, normalize_tot_weights=False, am_beta=1.0,
              weight=0.5, no_transition_cost=NTC)          # exp/wsj/decode.sh
FLAGS = [dict(normalize_am_weights=a, normalize_lm_weights=l, normalize_tot_weights=t)
         for a in (True, False) for l in (True, False) for t in (True, False)]


@pytest.fixture(autouse=True)
def _memo_rows(monkeypatch):
    monkeypatch.setattr(LO, "costs_row", F.memo_rows)


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _lm_file(tmp_path, V, S, start, arcs, arc_type="standard"):
    path = str(tmp_path / ("lm_%d_%s.fst" % (V, arc_type)))
    cmap = F.write(path, V, S, start, arcs, arc_type=arc_type)
    return path, cmap, F.memo(LO.from_tables(package().lm.load(path, cmap, V)))


def _rec(V, path, cmap, cfg=None, **o):
    cfg = cfg or O.make_config(**dict(PYRAMID, num_phonemes=V))
    return make_recognizer(cfg, O.init_params(cfg, seed=1), lm=dict(DECODE, path=path, **o), character_map=cmap)


def _canon(sets):
    """[n] dicts -> states int [n, 7] sorted with -1 padding, weights float64 [n, 7] (0 in the padding)."""
    st = np.full((len(sets), LO.MAX_STATES), -1, np.int64)
    wt = np.zeros((len(sets), LO.MAX_STATES))
    for i, s in enumerate(sets):
        for j, k in enumerate(sorted(s)):
            st[i, j], wt[i, j] = k, s[k]
    return st, wt


def _check(st, sets, rows, errs, row_idx=None):
    """Every row of the device state `st` against the oracle's sets (the same states, weights to 1e-9 relative, floor
    1) and the rows `row_idx` (default: all) against its cost rows `rows` (rtol = atol = 1e-5).  errs: worst errors
    so far."""
    gs = st["lm_states"].cpu().numpy().astype(np.int64)
    gw = st["lm_weights"].cpu().numpy()
    ga = st["lm_add"].cpu().numpy()
    if row_idx is not None:
        ga = ga[row_idx]
    order = np.argsort(np.where(gs < 0, np.iinfo(np.int64).max, gs), axis=1, kind="stable")
    gs, gw = np.take_along_axis(gs, order, 1), np.take_along_axis(gw, order, 1)
    ws, ww = _canon(sets)
    bad = np.flatnonzero((gs != ws).any(1))
    assert not bad.size, ("states differ", bad[:4], gs[bad[:2]], ws[bad[:2]])
    we = np.abs(gw - ww) / np.maximum(1.0, np.abs(ww))
    want = np.stack(rows).astype(np.float64)
    ae = np.abs(ga.astype(np.float64) - want)
    assert we.max() <= SET_TOL, ("weights", we.max(), np.unravel_index(we.argmax(), we.shape))
    assert (ae <= ROW_TOL + ROW_TOL * np.abs(want)).all(), ("rows", ae.max(), np.unravel_index(ae.argmax(), ae.shape))
    errs["set"] = max(errs.get("set", 0.0), float(we.max()))
    errs["row"] = max(errs.get("row", 0.0), float(ae.max()))
    errs["max_states"] = max(errs.get("max_states", 0), int((ws >= 0).sum(1).max()))
    errs["rows_ge3"] = errs.get("rows_ge3", 0) + int(((ws >= 0).sum(1) >= 3).sum())
    errs["weight_max"] = max(errs.get("weight_max", 0.0), float(np.abs(ww).max()))
    errs["finite_past_32"] = errs.get("finite_past_32", 0) + int((want[:, 32:] < NTC).sum())


def _walk(rec, fst, V, R, steps, seed, distinct=None, symbols=None, errs=None):
    """R rows along D = min(R, distinct) seeded symbol sequences (row r follows sequence r mod D) through
    _lm_initial_states / _lm_next_states, every row checked after every step.  The symbols are `symbols` [steps, D]
    if given, else one the set has a finite cost for, 9 times in 10."""
    D = R if distinct is None else min(R, distinct)
    rng = np.random.RandomState(seed)
    errs = {} if errs is None else errs
    st = rec._lm_initial_states(R)
    s0, row0 = LO.initial(fst, V, NTC)
    sets, rows = [dict(s0) for _ in range(D)], [row0] * D
    idx = np.arange(R) % D
    _check(st, [sets[i] for i in idx], [rows[i] for i in idx], errs)
    for t in range(steps):
        ys = []
        for row in rows:
            known = np.flatnonzero(row < np.float32(NTC))
            ys.append(int(rng.choice(known)) if known.size and rng.rand() < 0.9 else int(rng.randint(V)))
        ys = np.array(ys if symbols is None else symbols[t], np.int64)
        st = rec._lm_next_states(st, ys[idx])
        sets = [fst.advance(s, int(y) + 1) for s, y in zip(sets, ys)]
        rows = [fst.row(s, V, NTC) for s in sets]
        _check(st, [sets[i] for i in idx], [rows[i] for i in idx], errs)
    return errs


# ---- 1. vocabulary widths -----------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def ngrams(tmp_path_factory):
    d = tmp_path_factory.mktemp("ngrams")
    return {V: _lm_file(d, V, *F.ngram(V, seed=7)) for V in WIDTHS + [32]}


@pytest.mark.parametrize("V", WIDTHS)
def test_lm_states_at_every_width(ngrams, V):
    _torch()
    path, cmap, fst = ngrams[V]
    rec = _rec(V, path, cmap)
    errs = {}
    for R in (1, 3, 5, 4097):
        _walk(rec, fst, V, R, 10, seed=R, distinct=32, errs=errs)
    print("V", V, errs)
    assert errs["max_states"] >= 2
    if V > 32:                              # symbols of the lanes' second pass had finite costs
        assert errs["finite_past_32"] > 0


def _fused_case(V, path, cmap, fst, attention="content_and_conv", flags=FLAGS):
    M = CO if attention == "content" else O
    cfg = M.make_config(**dict(PYRAMID, num_phonemes=V))
    params = M.init_params(cfg, seed=4, scale=10.0)
    x, m, labels, lmask = O.synthetic_batch(cfg, B=3, T=40, seed=5)
    att, attm = O.encoder(cfg, params, x, m)
    r = M.cost_matrix(cfg, params, att, attm, labels, lmask, return_all=True)
    logits = O.readout(cfg, params, r["states"], r["weighted_averages"])
    content = attention == "content"
    pkg = package()
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": cfg["num_features"]}, input_num_chars={}, eos_label=cfg["eos_label"],
        num_phonemes=V, dim_dec=cfg["dim_dec"], dims_bidir=cfg["dims_bidir"], subsample=cfg["subsample"],
        conv_n=None if content else cfg["conv_n"], conv_num_filters=1 if content else cfg["conv_num_filters"],
        dim_matcher=cfg["dim_matcher"], post_merge_dims=cfg["post_merge_dims"],
        post_merge_activation=pkg.Maxout(cfg["maxout_pieces"]), dim_output_embedding=cfg["dim_feedback"],
        prior=None if content else cfg["prior"], attention_type=attention, enc_transition=pkg.GatedRecurrent,
        dec_transition=pkg.GatedRecurrent, data_prepend_eos=False, lm=dict(DECODE, path=path), character_map=cmap)
    rec.set_parameter_values(params)
    lib, h = pkg._lib.load(), rec._require_ready()
    gatt, gattm = rec.encode(x, m)
    add = LO.lm_path(fst, labels, lmask, V, NTC)
    worst = 0.0
    for fl in flags:
        for am_beta, weight in ((1.0, 0.5), (0.7, 1.0)):
            o = dict(fl, am_beta=am_beta, weight=weight, no_transition_cost=NTC)
            rec.lm.update(o)
            rec._attach_lm(lib, h)
            got = rec.cost_matrix(labels, lmask, gatt, gattm).cpu().numpy().astype(np.float64)
            want = np.take_along_axis(LO.fused_costs(logits, add, o), labels[..., None], axis=-1)[..., 0] * lmask
            assert np.allclose(got, want, rtol=FUSED_TOL, atol=FUSED_TOL), (o, np.abs(got - want).max())
            worst = max(worst, float(np.abs(got - want).max()))
    return worst, labels, add


@pytest.mark.parametrize("V", WIDTHS)
def test_fused_cost_matrix_at_every_width(ngrams, V):
    _torch()
    path, cmap, fst = ngrams[V]
    worst, labels, add = _fused_case(V, path, cmap, fst)
    print("V", V, "worst fused cost error %.2e" % worst)
    if V > 32:
        assert (add[..., 32:] < NTC).any()       # the readout's rows past 32 carried finite LM costs


@pytest.mark.parametrize("V,decoder,attention", [(63, "stepwise", "content_and_conv"), (65, "persistent", "content")])
def test_fused_cost_matrix_decoders_and_attention(ngrams, V, decoder, attention, monkeypatch):
    _torch()
    if decoder == "stepwise":
        monkeypatch.setenv("LVSR_NO_DEC_SCAN", "1")
    path, cmap, fst = ngrams[V]
    worst, _, _ = _fused_case(V, path, cmap, fst, attention=attention)
    print(V, decoder, attention, "worst fused cost error %.2e" % worst)


def test_vocabulary_above_128_is_refused(ngrams, tmp_path):
    """lvsr_model_create accepts 1 to 128 symbols, lm_step's range, so no LM kernel ever meets a wider row."""
    _torch()
    path, cmap, fst = ngrams[128]
    rec = _rec(128, path, cmap)
    before = rec._lm_initial_states(3)
    p129, cmap129, _ = _lm_file(tmp_path, 129, *F.ngram(129, seed=7))
    cfg = O.make_config(**dict(PYRAMID, num_phonemes=129))
    big = make_recognizer(cfg, lm=dict(DECODE, path=p129), character_map=cmap129)
    with pytest.raises(RuntimeError, match="num_phonemes out of range"):
        big._require_ready()
    again = rec._lm_initial_states(3)
    for k in before:
        assert np.array_equal(before[k].cpu().numpy(), again[k].cpu().numpy())


# ---- 2. set sizes and closure caps --------------------------------------------------------------------------------

def test_set_sizes_and_closure_caps(tmp_path):
    torch = _torch()
    V = 32
    S, start, arcs, info = F.limits_fst(V, seed=3)
    path, cmap, fst = _lm_file(tmp_path, V, S, start, arcs)
    rec = _rec(V, path, cmap)
    init = rec._lm_initial_states(10)
    s0, row0 = LO.initial(fst, V, NTC)
    errs = {}
    _check(init, [s0] * 10, [row0] * 10, errs)
    y = lambda v: torch.tensor(v, dtype=torch.int64)

    def good():
        """sets of 1..7 states, gateway P (a candidate with a 32-state closure) and the start again"""
        return rec._lm_next_states(init, y([0, 1, 2, 3, 4, 5, 6, 8, 8, 0]))

    ref = good()
    want = [fst.advance(s0, c + 1) for c in (0, 1, 2, 3, 4, 5, 6, 8, 8, 0)]
    _check(ref, want, [fst.row(s, V, NTC) for s in want], errs)
    assert [len(s) for s in want[:7]] == list(range(1, 8)) and errs["max_states"] == 7
    P = want[7]
    assert len(fst.advance(P, 1)) == F.CLOSURE_OK and ref["lm_add"][7, 0].item() < NTC

    def same():
        again = good()
        for k in ref:
            assert torch.equal(again[k], ref[k]), k

    # each refusal advances one row, so that its error is the only one the status word can hold
    start1 = {k: v[:1] for k, v in init.items()}
    with pytest.raises(ValueError, match="outputs"):
        rec._lm_next_states(init, y([7]))                     # one symbol for 10 rows
    same()
    with pytest.raises(RuntimeError, match="more than 7"):
        rec._lm_next_states(start1, y([7]))                   # 8 states
    same()
    with pytest.raises(RuntimeError, match="more than 7"):
        rec._lm_next_states({k: v[7:8] for k, v in ref.items()}, y([0]))    # P's 32-state closure taken: 32 states
    same()
    with pytest.raises(RuntimeError, match="epsilon closure exceeded 32"):
        rec._lm_next_states(start1, y([9]))                   # {Q}: its cost row meets the 33-state closure
    same()
    q_states = torch.full((1, LO.MAX_STATES), -1, dtype=torch.int32, device=rec.device)
    q_states[0, 0] = info["Q"]
    q = dict(lm_states=q_states, lm_weights=torch.zeros((1, LO.MAX_STATES), dtype=torch.float64, device=rec.device))
    with pytest.raises(RuntimeError, match="epsilon closure exceeded 32"):
        rec._lm_next_states(q, y([0]))                        # the 33-state closure as the taken transition
    same()
    print("set sizes 1-7 and the 32-state candidate:", errs)


# ---- 3. closure order and mixed-sign weights ----------------------------------------------------------------------

@pytest.mark.parametrize("arc_type", ["standard", "log"])
def test_closure_order_and_mixed_sign_weights(tmp_path, arc_type):
    _torch()
    V = 32
    S, start, arcs = F.order_fst(V, seed=11)
    path, cmap, fst = _lm_file(tmp_path, V, S, start, arcs, arc_type=arc_type)
    rec = _rec(V, path, cmap)
    errs = _walk(rec, fst, V, 130, 16, seed=4)
    print(arc_type, errs)
    assert errs["max_states"] == 7


# ---- 4. long walks ------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def four_gram():
    return F.four_gram()


@pytest.mark.parametrize("variant", ["plain", "pushed"])
def test_long_walks_on_the_four_gram(tmp_path, four_gram, variant):
    _torch()
    V, S, start, arcs = four_gram
    if variant == "pushed":
        arcs = F.pushed(S, arcs, seed=1)
    path, cmap, fst = _lm_file(tmp_path, V, S, start, arcs)
    rec = _rec(V, path, cmap)
    W = F.LONG_WALK           # the walk tests/test_lm_matrix_cpu.py restates in float32
    errs = _walk(rec, fst, V, W["rows"], W["steps"], 0, symbols=F.uniform_walk(V, **W))
    print(variant, errs)
    # set weights in the hundreds: a cost is the difference of two such sums (float32 would miss by 1e-5 and more)
    assert errs["max_states"] == 4 and errs["weight_max"] > 300


# ---- 5. teacher forcing with masks --------------------------------------------------------------------------------

def _forced_labels(fst, V, L, B, seed):
    """Labels the LM knows (9 times in 10) and masks: ragged lengths, zeros in the middle of some rows (with symbols
    there that would change the set), one row masked entirely."""
    rng = np.random.RandomState(seed)
    labels = np.zeros((L, B), np.int64)
    mask = np.zeros((L, B), np.float32)
    for b in range(B):
        n = L if b % 4 == 0 else int(rng.randint(1, L + 1))
        mask[:n, b] = 1
        if b % 3 == 1 and n > 4:
            lo = int(rng.randint(1, n - 2))
            mask[lo:lo + int(rng.randint(1, min(8, n - lo))), b] = 0
        s, row = LO.initial(fst, V, NTC)
        for i in range(L):
            known = np.flatnonzero(row < np.float32(NTC))
            labels[i, b] = rng.choice(known) if known.size and rng.rand() < 0.9 else rng.randint(V)
            if mask[i, b]:
                s = fst.advance(s, int(labels[i, b]) + 1)
                row = fst.row(s, V, NTC)
    mask[:, B // 2] = 0
    return labels, mask


@pytest.mark.parametrize("L", [300, 1])
def test_teacher_forcing_with_masks(ngrams, L):
    _torch()
    V, B = 32, 64
    path, cmap, fst = ngrams[V]
    cfg = O.make_config(**dict(PYRAMID, num_phonemes=V))
    params = O.init_params(cfg, seed=4, scale=10.0)
    x, m, _, _ = O.synthetic_batch(cfg, B=B, T=48, seed=5)
    labels, lmask = _forced_labels(fst, V, L, B, seed=6)
    assert L == 1 or ((lmask[:-1] == 0) & (lmask[1:] == 1)).any()   # zeros in the middle of a row
    rec = make_recognizer(cfg, params, lm=dict(DECODE, path=path), character_map=cmap)
    lib, h = package()._lib.load(), rec._require_ready()
    gatt, gattm = rec.encode(x, m)
    add = LO.lm_path(fst, labels, lmask, V, NTC)
    # am_beta 0, weight 1, no normalisation: the fused cost is the LM row's entry at the label
    rec.lm.update(dict(normalize_am_weights=False, normalize_lm_weights=False, normalize_tot_weights=False, am_beta=0.0,
                       weight=1.0))
    rec._attach_lm(lib, h)
    got = rec.cost_matrix(labels, lmask, gatt, gattm).cpu().numpy().astype(np.float64)
    want = np.take_along_axis(add, labels[..., None], axis=-1)[..., 0].astype(np.float64) * lmask
    e_add = float(np.abs(got - want).max())
    assert np.allclose(got, want, rtol=ROW_TOL, atol=ROW_TOL), e_add
    assert not got[:, B // 2].any()
    # and through the fused readout at decode.sh's and the lm-normalised settings
    att, attm = O.encoder(cfg, params, x, m)
    r = O.cost_matrix(cfg, params, att, attm, labels, lmask, return_all=True)
    logits = O.readout(cfg, params, r["states"], r["weighted_averages"])
    worst = 0.0
    for o in (DECODE, dict(DECODE, normalize_lm_weights=True)):
        rec.lm.update(o)
        rec._attach_lm(lib, h)
        got = rec.cost_matrix(labels, lmask, gatt, gattm).cpu().numpy().astype(np.float64)
        want = np.take_along_axis(LO.fused_costs(logits, add, o), labels[..., None], axis=-1)[..., 0] * lmask
        assert np.allclose(got, want, rtol=FUSED_TOL, atol=FUSED_TOL), np.abs(got - want).max()
        worst = max(worst, float(np.abs(got - want).max()))
    print("L", L, "LM column error %.2e, fused %.2e" % (e_add, worst))


# ---- 6. the million-arc 4-gram with a wide start state ------------------------------------------------------------

def test_wide_four_gram_at_the_search_row_count(tmp_path, four_gram):
    _torch()
    V, S, start, arcs = four_gram
    S2, W, arcs2 = F.wide(V, S, arcs, seed=3)
    path, cmap, fst = _lm_file(tmp_path, V, S2, W, arcs2)
    rec = _rec(V, path, cmap)
    t0 = time.time()
    R, steps = 6400, 50
    ys = F.uniform_walk(V, R, steps, seed=9)                 # 6,400 independent walks
    pick = np.random.RandomState(10)
    st = rec._lm_initial_states(R)
    s0, row0 = LO.initial(fst, V, NTC)
    sets, errs = [s0] * R, {}
    _check(st, sets, [row0] * R, errs)
    for t in range(steps):
        st = rec._lm_next_states(st, ys[t])
        # every row's set; the cost rows of a fresh seeded sample of 256 rows (a row costs the oracle 33 advances)
        sets = [LO.FST.advance(fst, s, int(y) + 1) for s, y in zip(sets, ys[t])]
        idx = np.sort(pick.choice(R, 256, replace=False))
        _check(st, sets, [fst.row(sets[i], V, NTC) for i in idx], errs, row_idx=idx)
    print("6400 rows x 50 steps:", errs, "%.1f s" % (time.time() - t0))
    assert errs["max_states"] == 7 and errs["rows_ge3"] > R * 40


# ---- 7. the fused search at the benchmark's shape -------------------------------------------------------------------

def test_fused_search_at_the_bench_shape(tmp_path, four_gram, monkeypatch):
    """bench.py's configs[2] network and weights, 32 utterances x 800 frames, the 4-gram at decode.sh's settings
    (weight 0.5, no_transition_cost 20, char_discount 1.0).  Beam 10: the tokens of every utterance whose float64
    search meets a gap of at least 1e-3 at each k boundary equal O.beam_search's, over a search of 30 steps or more.
    Beam 200: every hypothesis' cumulative costs equal the teacher-forced oracle of its own tokens.

    The best hypotheses stay short (mean length about 1): with this synthetic model no eos bias makes them long at
    decode.sh's settings, as a symbol costs more than the char discount of 1.0 gives back (DESIGN.md §1)."""
    _torch()
    V, S, start, arcs = four_gram
    path, cmap, fst = _lm_file(tmp_path, V, S, start, arcs)
    cfg = O.make_config(max_decoded_length_scale=8.0, **bench.NET)
    rec = make_recognizer(cfg, lm=dict(DECODE, path=path), character_map=cmap)
    params = bench.search_values(rec.parameter_shapes())
    rec.set_parameter_values(params)
    p32 = {k: f32(v) for k, v in params.items()}
    rng = np.random.RandomState(99)
    utts = [rng.normal(size=(800, 40)).astype(np.float32) for _ in range(32)]
    maxl = [int(800 / 8.0)] * 32
    t0 = time.time()
    rec.init_beam_search(10)
    got = rec._beam_search.search_many(utts, cfg["eos_label"], maxl, raise_on_failure=False, char_discount=1.0)
    lengths = [len(g[0][0]) for g in got if g is not None]
    print("beam 10: decoded %d of 32, mean best length %.2f" % (len(lengths), np.mean(lengths)))
    assert len(lengths) >= 20

    gaps = []
    O_smallest = O.smallest

    def smallest(matrix, k):
        flat = np.sort(matrix.reshape(-1))
        if flat.shape[0] > k:
            gaps.append(flat[k] - flat[k - 1])
        return O_smallest(matrix, k)

    monkeypatch.setattr(O, "smallest", smallest)
    comp = LO.computers(cfg, p32, fst, DECODE)
    compared, worst, tried, steps, lens10 = 0, 0.0, 0, [], []
    for x, g in zip(utts, got):
        if compared >= 5 or tried >= 12:
            break
        tried += 1
        att, attm = rec.encode(x[:, None, :])
        ctx = (att.double().cpu().numpy(), attm.double().cpu().numpy())
        del gaps[:]
        stats = {}
        try:
            want = O.beam_search(cfg, p32, x, 10, char_discount=1.0, computers=dict(comp, context=lambda r: ctx),
                                 stats=stats)
        except O.CandidateNotFoundError:
            want = None
        if min(gaps) < 1e-3:
            continue
        compared += 1
        steps.append(stats["steps"])
        if want is None:
            assert g is None
            continue
        assert g is not None and g[0] == want[0]
        worst = max(worst, elementwise_err(g[1], want[1]))
        lens10 += [len(t) for t in want[0]]
    monkeypatch.setattr(O, "smallest", O_smallest)
    print("beam 10: compared %d of %d utterances tried over %s steps, %d finished hypotheses of %s symbols, worst "
          "total cost error %.2e" % (compared, tried, steps, len(lens10), sorted(set(lens10)), worst))
    assert compared >= 4 and min(steps) >= 30 and worst <= SEARCH_COST_TOL

    rec.init_beam_search(200)
    three = utts[:3]
    got = rec._beam_search.search_many(three, cfg["eos_label"], maxl[:3], as_arrays=True, raise_on_failure=False,
                                       char_discount=1.0)
    worst, n = _anchor(rec, cfg, params, three, got,
                       lambda a, m, y, ym: LO.cost_matrix(cfg, p32, fst, DECODE, a, m, y, ym))
    lens = np.array([int(k) for r in got if r is not None for k in r[1].sum(0)])
    print("beam 200: hypotheses %d of %s symbols (mean %.1f), worst cumulative cost error %.2e, %.1f s"
          % (n, np.bincount(lens).nonzero()[0].tolist(), lens.mean(), worst, time.time() - t0))
    assert n >= 30 and n == lens.size and worst <= SEARCH_COST_TOL
