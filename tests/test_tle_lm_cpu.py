"""Task loss estimation with an FST language model on the host: the float64 oracle of tests/tle_lm_oracle.py pinned
against the TLE and LM oracles it composes and against two cases worked by hand, and the refusals that remain (training
a TLE + LM model, sampling a log-likelihood model with an LM)."""
import sys

import numpy as np
import pytest

import lm_oracle as LO
import tle_lm_oracle as TLO
import tle_oracle as TO
from compat_helpers import COMPAT, write_experiment
from helpers import O, package

NET = dict(num_features=12, dims_bidir=[16], subsample=[1], dim_dec=16, dim_matcher=16, conv_n=3, conv_num_filters=4,
           num_phonemes=9, post_merge_dims=[16], maxout_pieces=2)
OFF = dict(normalize_am_weights=False, normalize_lm_weights=False, normalize_tot_weights=False)


@pytest.fixture(scope="module")
def model():
    cfg = O.make_config(**NET)
    params = O.init_params(cfg, seed=3, scale=10.0)
    x, m, labels, lmask = O.synthetic_batch(cfg, B=3, T=14, seed=4)
    att, attm = O.encoder(cfg, params, x, m)
    S, start, arcs = LO.char_ngram(cfg["num_phonemes"], seed=5, n_tri=6)
    return cfg, params, att, attm, labels, lmask, LO.FST(S, start, arcs)


@pytest.mark.parametrize("name", ["mse_gain", "mse_reward"])
@pytest.mark.parametrize("ntc", [20.0, 1e12])
def test_weight_zero_without_normalisation_is_the_tle_oracle(model, name, ntc):
    cfg, params, att, attm, labels, lmask, fst = model
    crit = dict(name=name, min_reward=-5.0)
    o = dict(OFF, weight=0.0, am_beta=1.0, no_transition_cost=ntc)
    g = labels[::-1].copy()
    g[-1] = cfg["eos_label"]
    for gt in (None, g):
        got = TLO.cost_matrix(cfg, params, fst, o, att, attm, labels, lmask, crit, groundtruth=gt)
        want = TO.cost_matrix(cfg, params, att, attm, labels, lmask, crit, groundtruth=gt)
        np.testing.assert_array_equal(got, want)
    got_o, got_c, _ = TLO.generate_greedy(cfg, params, fst, o, att, attm, 6)
    want_o, want_c, _ = TO.generate_greedy(cfg, params, att, attm, 6)
    np.testing.assert_array_equal(got_o, want_o)
    np.testing.assert_array_equal(got_c, want_c)


def test_fused_rows_are_the_lm_oracles_on_the_tle_readouts(model):
    cfg, params, att, attm, labels, lmask, fst = model
    o = dict(normalize_am_weights=True, normalize_lm_weights=True, normalize_tot_weights=False, weight=0.3,
             am_beta=0.7, no_transition_cost=20.0)
    r = TLO.cost_matrix(cfg, params, fst, o, att, attm, labels, lmask, dict(name="mse_gain"), return_all=True)
    ro, _ = TO.readouts(cfg, params, att, attm, labels, lmask)
    np.testing.assert_array_equal(r["logits"], ro)
    np.testing.assert_array_equal(r["add"], LO.lm_path(fst, labels, lmask, cfg["num_phonemes"], 20.0))
    np.testing.assert_array_equal(-r["readouts"], LO.fused_costs(ro, r["add"], o))
    # the emitter costs of a search row are the same -x, the row the log-likelihood emitter writes under fusion
    B = att.shape[1]
    st = TLO.initial_states(cfg, params, fst, o, B, att)
    assert (st["outputs"] == 0).all()
    c = TLO.emitter_costs(cfg, params, o, att, attm, st)
    wa, _, _, _ = O.take_glimpses(cfg, params, att, None, attm, st["weights"], st["step"], st["states"])
    np.testing.assert_array_equal(c, LO.fused_costs(O.readout(cfg, params, st["states"], wa), st["lm_add"], o))
    np.testing.assert_array_equal(c, -TLO.fused_readouts(O.readout(cfg, params, st["states"], wa), st["lm_add"], o))


def test_greedy_generation_advances_the_lm_by_the_emitted_symbols(model):
    cfg, params, att, attm, labels, lmask, fst = model
    o = dict(OFF, normalize_am_weights=True, weight=0.8, am_beta=1.0, no_transition_cost=20.0)
    outs, costs, st = TLO.generate_greedy(cfg, params, fst, o, att, attm, 5)
    V = cfg["num_phonemes"]
    for b in range(att.shape[1]):
        s, _ = LO.initial(fst, V, 20.0)
        for y in outs[:, b]:
            s, row = LO.next_state(fst, s, y, V, 20.0)
        assert st["lm_sets"][b] == s
        np.testing.assert_array_equal(st["lm_add"][b], row)
    # teacher forcing the generated outputs reproduces the emitted x as the picked fused readouts
    r = TLO.cost_matrix(cfg, params, fst, o, att, attm, outs, None, dict(name="mse_gain"), return_all=True)
    picked = np.take_along_axis(r["readouts"], outs[..., None], axis=-1)[..., 0]
    np.testing.assert_allclose(picked, costs, rtol=1e-12, atol=1e-12)


# V = 3, eos = 2; start state 0 --0/1.0--> 1 --2/0.5--> 2, 0 --1/2.0--> 2, no epsilon arcs; no_transition_cost 10.
# add = [[1, 2, 10], [10, 10, 0.5]] along the labels [0, 2].  With weight 0.5, am_beta 2 and no normalisation,
# x = 2 r - 0.5 add = [[1.5, -1, -7], [-4, -6, 3.75]] for r = [[1, 0, -1], [0.5, -0.5, 2]].
# Groundtruth = prediction = [0, 2]: R = [[0, -1, -1], [-1, -1, 0]], G = [[0, -1, -1], [-1, -1, 0]].
HAND_FST = LO.FST(3, 0, [[(1, 1, 1.0), (2, 2, 2.0)], [(3, 2, 0.5)], []])
HAND_O = dict(OFF, weight=0.5, am_beta=2.0, no_transition_cost=10.0)
HAND_R = np.array([[[1.0, 0.0, -1.0]], [[0.5, -0.5, 2.0]]])
HAND_Y = np.array([[0], [2]])


@pytest.mark.parametrize("name,want", [
    ("mse_gain", [1.5 ** 2 + 0 + 6.0 ** 2, 3.0 ** 2 + 5.0 ** 2 + 3.75 ** 2]),                # G >= min_reward = -1
    # predicted = x + cumsum of the picked x with the first step's zeroed: step 1 adds x[1, 2] = 3.75
    ("mse_reward", [1.5 ** 2 + 0 + 6.0 ** 2, 0.75 ** 2 + 1.25 ** 2 + 7.5 ** 2]),
])
def test_hand_worked_case(name, want):
    cfg = dict(num_phonemes=3, eos_label=2)
    add = LO.lm_path(HAND_FST, HAND_Y, None, 3, 10.0)
    np.testing.assert_array_equal(add[:, 0], [[1, 2, 10], [10, 10, 0.5]])
    x = TLO.fused_readouts(HAND_R, add, HAND_O)
    np.testing.assert_allclose(x[:, 0], [[1.5, -1, -7], [-4, -6, 3.75]], rtol=0, atol=1e-12)
    got = TLO.cost_of_logits(cfg, HAND_FST, HAND_O, dict(name=name, min_reward=-1.0), HAND_R, HAND_Y)
    np.testing.assert_allclose(got[:, 0], want, rtol=1e-12)


def _small_lm(tmp_path):
    V = 6
    S, start, arcs = LO.char_ngram(V, seed=3, n_tri=5)
    path = str(tmp_path / "lm.fst")
    return path, LO.to_file(path, V, S, start, arcs, seed=1)


def _kw(**extra):
    kw = dict(input_dims={"recordings": 40}, input_num_chars={}, eos_label=1, num_phonemes=6, dim_dec=8,
              dims_bidir=[8], conv_n=1, post_merge_dims=[8])
    kw.update(extra)
    return kw


def test_tle_with_an_lm_builds_and_only_training_is_refused(tmp_path):
    pkg = package()
    path, cmap = _small_lm(tmp_path)
    lm = dict(path=path, weight=0.15)                      # decode_tle.sh's overrides; the rest at their defaults
    rec = pkg.SpeechRecognizer(**_kw(lm=lm, character_map=cmap, criterion=dict(name="mse_reward")))
    assert rec.tle and rec.lm["weight"] == 0.15 and rec.lm["normalize_am_weights"] is True
    assert rec.lm["normalize_lm_weights"] is False and rec.lm["normalize_tot_weights"] is False
    with pytest.raises(NotImplementedError, match="language model"):
        pkg.GradientDescent(recognizer=rec)
    with pytest.raises(NotImplementedError, match="language model"):
        pkg.GradientDescent(recognizer=rec, exploration="greedy")
    import pickle
    back = pickle.loads(pickle.dumps(rec))
    assert back.criterion == rec.criterion and back.lm == rec.lm and back._lm_tables["num_states"] > 0
    # a log-likelihood model with an LM still does not sample: LMEmitter.emit returns zeros in the reference
    ll = pkg.SpeechRecognizer(**_kw(lm=lm, character_map=cmap))
    with pytest.raises(NotImplementedError, match="language model"):
        ll.sample({"recordings": np.zeros((10, 40), np.float32)})


def test_compat_train_refuses_a_tle_model_with_an_lm(tmp_path, monkeypatch):
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as C
    import lvsr.main as main
    exp = write_experiment(tmp_path)
    chars = list("abcdefghijk") + ["$"]
    S, start, arcs = LO.char_ngram(len(chars), seed=1, n_tri=8)
    fst_path = str(tmp_path / "lm.fst")
    LO.to_file(fst_path, len(chars), S, start, arcs, seed=3)
    with open(fst_path, "rb") as f:                      # the data's characters as the FST's input symbols
        blob = f.read()
    for k in reversed(range(len(chars))):
        old, new = ("c%d" % k).encode(), chars[k].encode()
        blob = blob.replace(len(old).to_bytes(4, "little") + old, len(new).to_bytes(4, "little") + new)
    with open(fst_path, "wb") as f:
        f.write(blob)
    cfg = C.Configuration(exp["base"], None, [("net.criterion", "{name: mse_gain, min_reward: -5}"),
                                              ("net.lm.path", repr(fst_path)), ("net.lm.weight", "0.15")])
    built = []

    def create_model(config, data, params):              # the recognizer as compat builds it, without its device
        net = dict(config["net"])
        rec = main.pkg.SpeechRecognizer(input_dims={"recordings": data.num_features}, input_num_chars={},
                                        eos_label=data.eos_label, num_phonemes=data.num_labels,
                                        data_prepend_eos=data.prepend_eos, character_map=data.character_map, **net)
        built.append(rec)
        return rec
    monkeypatch.setattr(main, "create_model", create_model)
    with pytest.raises(NotImplementedError, match="language model"):
        main.train(cfg, str(tmp_path / "model"))
    assert built and built[0].tle and built[0].lm["weight"] == 0.15
