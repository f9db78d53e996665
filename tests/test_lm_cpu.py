"""Host side of LM shallow fusion: the OpenFST reader and the arc table it builds, the oracle's FST operations on a
hand-built FST with answers computed by hand, the recognizer's refusals and the compat character map."""
import math
import sys

import numpy as np
import pytest

import lm_oracle as LO
from helpers import package


def _lm():
    return package().lm


def _small_file(tmp_path, **kw):
    V = 6
    S, start, arcs = LO.char_ngram(V, seed=3, n_tri=5)
    path = str(tmp_path / "lm.fst")
    cmap = LO.to_file(path, V, S, start, arcs, seed=1) if not kw else None
    return path, cmap, V, S, start, arcs


def test_reader_round_trip_and_arc_table(tmp_path):
    path, cmap, V, S, start, arcs = _small_file(tmp_path)
    t = _lm().load(path, cmap, V)
    assert t["num_states"] == S and t["start"] == start and t["offsets"][-1] == sum(len(a) for a in arcs)
    got = LO.from_tables(t)
    for s in range(S):
        want = sorted((lab, nx, float(np.float32(w))) for lab, nx, w in arcs[s])
        assert sorted(got.arcs[s]) == want
        labs = [(l, n) for l, n, _ in got.arcs[s]]
        assert labs == sorted(labs)                        # sorted by (label, next state)
    # another character map permutes the NN labels
    rev = {ch: V - 1 - i for ch, i in cmap.items()}
    t2 = _lm().load(path, rev, V)
    a0 = sorted(LO.from_tables(t2).arcs[0])
    assert a0 == sorted((0 if l == 0 else V - l + 1, n, w) for l, n, w in got.arcs[0])


def _write(tmp_path, **kw):
    path = str(tmp_path / "x.fst")
    isyms = kw.pop("isyms", {"<eps>": 0, "a": 1, "b": 2})
    LO.write_fst(path, 2, 0, [[(1, 1, 0.5, 1)], []], isyms, **kw)
    return path


@pytest.mark.parametrize("kw,match", [(dict(magic=1234), "magic"), (dict(fst_type="const"), "FST type"),
                                      (dict(arc_type="log64"), "arc type"), (dict(isyms=None), "input symbol table")])
def test_reader_refusals(tmp_path, kw, match):
    with pytest.raises(ValueError, match=match):
        _lm().read_fst(_write(tmp_path, **kw))


def test_log_arcs_and_output_symbols_are_read(tmp_path):
    fst = _lm().read_fst(_write(tmp_path, arc_type="log", osyms={"<eps>": 0, "x": 1}))
    assert fst["isyms"] == {"<eps>": 0, "a": 1, "b": 2} and len(fst["arcs"][0]) == 1 and fst["arcs"][0]["nextstate"][0] == 1


def test_symbol_count_must_equal_the_character_map(tmp_path):
    path = _write(tmp_path)
    with pytest.raises(ValueError, match="input symbols"):
        _lm().load(path, {"a": 0, "b": 1, "c": 2}, 3)
    t = _lm().load(path, {"a": 1, "b": 0}, 2)
    assert list(t["label"]) == [2]                         # 'a' is NN label 1 -> arc label 2


# hand-built FST in NN space (labels: 1 = a, 2 = b, 0 = epsilon)
#   0 -a/1-> 1, 0 -a/2-> 2, 0 -b/3-> 4, 1 -eps/0.5-> 3, 2 -eps/0.25-> 3, 3 -eps/1-> 4, 3 -b/0.75-> 1
HAND = LO.FST(5, 0, [[(1, 1, 1.0), (1, 2, 2.0), (2, 4, 3.0)], [(0, 3, 0.5)], [(0, 3, 0.25)], [(0, 4, 1.0), (2, 1, 0.75)], []])


def _lsum(*xs):
    return -math.log(sum(math.exp(-x) for x in xs))


def test_transition_expand_and_costs_known_answers():
    assert HAND.transition({0: 0.0}, 1) == {1: 1.0, 2: 2.0}
    s = HAND.expand({1: 1.0, 2: 2.0})
    w3 = _lsum(1.5, 2.25)
    assert set(s) == {1, 2, 3, 4}
    assert math.isclose(s[3], w3, rel_tol=1e-12) and math.isclose(s[4], w3 + 1.0, rel_tol=1e-12)
    # a closure that reaches a state of the set it starts from: own weight and incoming paths are log-added
    s = HAND.expand({1: 0.2, 3: 0.4})
    assert math.isclose(s[3], _lsum(0.4, 0.7), rel_tol=1e-12) and math.isclose(s[4], s[3] + 1.0, rel_tol=1e-12)
    row = LO.costs_row(HAND, {0: 0.0}, 2, 20.0)
    assert row.dtype == np.float32
    assert row[0] == np.float32(_lsum(1.0, 2.0, w3, w3 + 1.0))
    assert row[1] == np.float32(3.0)
    # from {4} nothing leads anywhere; the empty set stays empty
    assert list(LO.costs_row(HAND, {4: 1.0}, 2, 20.0)) == [20.0, 20.0]
    assert HAND.advance({4: 1.0}, 1) == {} and list(LO.costs_row(HAND, {}, 2, 1e12)) == [np.float32(1e12)] * 2
    # b from {3, 4}: 3 -b-> 1, then 1 -eps-> 3 -eps-> 4
    s = HAND.advance({3: 0.0, 4: 0.0}, 2)
    assert s == pytest.approx({1: 0.75, 3: 1.25, 4: 2.25}, rel=1e-12)


def test_epsilon_cycles_and_large_sets_are_errors():
    cyc = LO.FST(3, 0, [[(0, 1, 1.0)], [(0, 2, 1.0)], [(0, 1, 1.0)]])
    with pytest.raises(LO.CycleError):
        cyc.expand({0: 0.0})
    loop = LO.FST(1, 0, [[(0, 0, 1.0)]])
    with pytest.raises(LO.CycleError):
        loop.expand({0: 0.0})
    wide = LO.FST(10, 0, [[(1, s, 1.0) for s in range(1, 10)]] + [[] for _ in range(9)])
    with pytest.raises(ValueError, match="more than 7"):
        LO.next_state(wide, {0: 0.0}, 0, 1, 20.0)


def _kw(**extra):
    kw = dict(input_dims={"recordings": 40}, input_num_chars={}, eos_label=1, num_phonemes=6, dim_dec=8,
              dims_bidir=[8], conv_n=1, post_merge_dims=[8])
    kw.update(extra)
    return kw


def test_recognizer_lm_refusals_and_config(tmp_path):
    pkg = package()
    with pytest.raises(NotImplementedError):                      # LMEmitter with the unfused readout
        pkg.SpeechRecognizer(**_kw(lm={"weight": 0.5}))
    with pytest.raises(NotImplementedError):                      # no way to map the symbols
        pkg.SpeechRecognizer(**_kw(lm={"path": "x.fst"}))
    path, cmap, V, S, start, arcs = _small_file(tmp_path)
    with pytest.raises(TypeError, match="unknown lm"):
        pkg.SpeechRecognizer(**_kw(lm={"path": path, "wieght": 0.5}, character_map=cmap))
    with pytest.raises(ValueError, match="symbols"):
        pkg.SpeechRecognizer(**_kw(lm={"path": path}, character_map={"c0": 0}))
    lm = {"path": path, "weight": 0.5, "no_transition_cost": 20}
    rec = pkg.SpeechRecognizer(**_kw(lm=lm, character_map=cmap))
    assert lm == {"path": path, "weight": 0.5, "no_transition_cost": 20}     # the caller's dict is not consumed
    assert rec.lm["weight"] == 0.5 and rec.lm["normalize_am_weights"] is True and rec.lm["am_beta"] == 1.0
    assert rec._lm_tables["num_states"] == S
    with pytest.raises(NotImplementedError):
        rec.sample({"recordings": np.zeros((10, 40), np.float32)})
    with pytest.raises(NotImplementedError):
        pkg.GradientDescent(recognizer=rec)
    import pickle
    back = pickle.loads(pickle.dumps(rec))
    assert back.lm == rec.lm and back._lm_tables["num_states"] == S
    assert np.array_equal(back._lm_tables["weight"], rec._lm_tables["weight"])


def test_compat_character_map(tmp_path):
    from compat_helpers import COMPAT, write_experiment
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    from lvsr.datasets import Data
    exp = write_experiment(tmp_path)
    data = Data(path=exp["npz"])
    chars = data.info_dataset.characters
    if chars is None:
        assert data.character_map is None
        z = dict(np.load(exp["npz"]))
        z["characters"] = np.array(["x%d" % i for i in range(int(z["num_labels"]))])
        np.savez(exp["npz"], **z)
        data = Data(path=exp["npz"])
        chars = data.info_dataset.characters
    assert data.character_map == {c: i for i, c in enumerate(chars)}
