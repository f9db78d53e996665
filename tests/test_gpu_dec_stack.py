"""The stacked decoder (net.dec_stack: 2) on the GPU against the float64 stack oracle (tests/stack_oracle.py): the
parameter table, the teacher-forced cost matrix with both layers' states, the BeamSearch state functions, greedy and
sampled generation, beam search one utterance at a time and in lock-step (with and without an FST language model),
and a Blocks checkpoint round trip.

The attention and the readout see the wide state rows [s0 | s1]; both layers step on decoder.cu's dense_kernel, layer 1
after layer 0, always step-wise (the persistent decoder holds one layer).  Element-wise bounds are
test_gpu_attention_plans.py's (DESIGN section 2): weights 5e-5 per element, energies 2e-5 of their scale, costs 1e-5,
states and weighted averages 1e-4, each with a floor of 0.1 of the tensor's scale.  The oracle decodes the GPU's own
encoder output, so the comparison measures the decoder alone.

Worst errors measured over this file on an H100 80GB HBM3 (700 W power limit): weights 1.3e-5, energies 2.4e-6, weight
sums 1.6e-7, costs 1.8e-6, states 6.7e-5 and weighted averages 2.4e-5 (both at dim_dec 512), search costs 7.0e-7."""
import ctypes
import os
import tarfile
from collections import OrderedDict

import numpy as np
import pytest

import lm_oracle as LO
import stack_oracle as SO
from helpers import O, elementwise_err, f32, package, rel_err
from test_gpu_attention_plans import TOL, _compare
from test_gpu_widths import _same_up_to_near_ties

pytestmark = pytest.mark.gpu

_ATT = "/recognizer/generator/att_trans/conv_att"
_RO = "/recognizer/generator/readout/post_merge/mlp/linear_0"

SMALL = dict(num_features=40, dims_bidir=[128], subsample=[1], dim_dec=128, dim_matcher=256, conv_n=8,
             conv_num_filters=10, num_phonemes=32, post_merge_dims=[128], maxout_pieces=2)
# wsj_jan_wsj13v2: 3 BiGRU(256), subsampling [1, 1, 2], one-of-N feedback, window around the mean
WSJ13V2 = dict(num_features=40, dims_bidir=[256, 256, 256], subsample=[1, 1, 2], dim_dec=256, dim_matcher=512,
               conv_n=100, conv_num_filters=10, num_phonemes=32, post_merge_dims=[256], maxout_pieces=2,
               embed_outputs=False, prior=dict(type="window_around_mean", before=150, after=150))
# wsj_jan_wsj15v2: the parent's 4 BiGRU(256), subsampling [1, 1, 2, 2], dim_dec 512
WSJ15V2 = dict(WSJ13V2, dims_bidir=[256, 256, 256, 256], subsample=[1, 1, 2, 2], dim_dec=512)
NARROW = dict(type="expanding", initial_begin=0, initial_end=6, min_speed=0.7, max_speed=2.2)
MEDIAN = dict(type="window_around_median", before=5, after=7)


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _recognizer(cfg, params=None, lm=None, cmap=None, dec_stack=2):
    pkg = package()
    content = cfg.get("attention_type") == "content"
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": cfg["num_features"]}, input_num_chars={}, eos_label=cfg["eos_label"],
        num_phonemes=cfg["num_phonemes"], dim_dec=cfg["dim_dec"], dims_bidir=cfg["dims_bidir"],
        subsample=cfg["subsample"], conv_n=None if content else cfg["conv_n"],
        conv_num_filters=cfg["conv_num_filters"], dim_matcher=cfg["dim_matcher"],
        post_merge_dims=cfg["post_merge_dims"], post_merge_activation=pkg.Maxout(cfg["maxout_pieces"]),
        dim_output_embedding=cfg["dim_feedback"] if cfg.get("embed_outputs", True) else None,
        embed_outputs=cfg.get("embed_outputs", True), prior=None if content else cfg["prior"],
        energy_normalizer=None if content else cfg["energy_normalizer"],
        attention_type="content" if content else "content_and_conv",
        max_decoded_length_scale=cfg["max_decoded_length_scale"], enc_transition=pkg.GatedRecurrent,
        dec_transition=pkg.GatedRecurrent, data_prepend_eos=False, lm=lm, character_map=cmap, dec_stack=dec_stack)
    if params is not None:
        rec.set_parameter_values(params)
    return rec


def _params(cfg, seed, gain=1.0, eos_bias=None):
    """Trained-like float32 parameters (scale 10) of the stack; gain / eos_bias sharpen the readout so that searches
    finish hypotheses within their length limit."""
    p = SO.init_params(cfg, seed=seed, scale=10.0)
    if cfg.get("energy_normalizer", "softmax") != "softmax" and cfg.get("attention_type") != "content":
        p[_ATT + "/energy_comp/linear.W"] *= 0.05             # energies in [2, 4], as test_gpu_attention_plans.py does
        p[_ATT + "/energy_comp/linear.b"][:] = 3.0
    p[_RO + ".W"] = p[_RO + ".W"] * gain
    if eos_bias is not None:
        p[_RO + ".b"][cfg["eos_label"]] = eos_bias
    return OrderedDict((k, f32(v)) for k, v in p.items())


def _encode(rec, cfg, B, T, seed):
    """The GPU encoder's output for a synthetic batch, as float64, with the labels and their mask."""
    x, m, labels, lm = O.synthetic_batch(cfg, B=B, T=T, seed=seed)
    att, attm = rec.encode(x, m)
    return att, attm, f32(att.cpu().numpy()), attm.cpu().numpy().astype(np.float64), x, m, labels, lm


def test_parameter_table_and_config_field():
    """The library's table is the oracle's at the wsj13v2 shape; a zero-filled dec_stack reads as 1, 3 is refused."""
    _torch()
    pkg = package()
    cfg = SO.make_config(**WSJ13V2)
    rec = _recognizer(cfg)
    assert list(rec.parameter_shapes().items()) == list(SO.param_shapes(cfg).items())
    single = _recognizer(O.make_config(**WSJ13V2), dec_stack=1)
    lib = pkg._lib.load()
    for value, want in ((0, single.parameter_shapes()), (3, None)):
        c = single._make_config()
        c.dec_stack = value
        h = ctypes.c_void_p()
        rc = lib.lvsr_model_create(ctypes.byref(c), ctypes.byref(h))
        if want is None:
            assert rc != 0 and b"dec_stack 3" in lib.lvsr_last_error()
            continue
        assert rc == 0
        try:
            names = [lib.lvsr_model_param_name(h, i).decode() for i in range(lib.lvsr_model_num_params(h))]
        finally:
            lib.lvsr_model_destroy(h)
        assert names == list(want)


COST_CASES = [
    ("wsj13v2", WSJ13V2, {}, 16, 80),
    ("wsj15v2_dim_dec512", WSJ15V2, {}, 37, 96),
    ("content_100rows", SMALL, dict(attention_type="content"), 100, 40),
    ("narrow_expanding", SMALL, dict(prior=NARROW), 37, 40),
    ("median", SMALL, dict(prior=MEDIAN), 16, 40),
    ("logistic_100rows", SMALL, dict(prior=MEDIAN, energy_normalizer="logistic"), 100, 32),
]


@pytest.mark.parametrize("case,arch,extra,B,T", COST_CASES, ids=[c[0] for c in COST_CASES])
def test_cost_matrix_matches_oracle(case, arch, extra, B, T):
    """Costs, weights, energies, both layers' states and the glimpses of cost_matrix; the decoder plan is step-wise."""
    torch = _torch()
    cfg = SO.make_config(**dict(arch, **extra))
    params = _params(cfg, seed=3)
    rec = _recognizer(cfg, params)
    att, attm, att64, attm64, x, m, labels, lm = _encode(rec, cfg, B, T, seed=5)
    got = rec.cost_matrix(labels, lm, att, attm, return_all=True)
    torch.cuda.synchronize()
    want = SO.cost_matrix(cfg, params, att64, attm64, labels, lm, return_all=True)
    assert tuple(got["states"].shape) == (labels.shape[0], B, 2 * cfg["dim_dec"])
    _compare(got, want, cfg.get("attention_type") == "content", case)
    plan = rec.decoder_plan()
    assert not plan["ran"] and plan["kernel"] == "stepwise", plan
    if case == "wsj13v2":
        # the host entry point (encoder + decoder, lvsr_recognizer_cost_host) against the whole float64 model
        assert rel_err(rec.cost(x, m, labels, lm), SO.recognizer_cost(cfg, params, x, m, labels, lm)) < 1e-4


@pytest.mark.parametrize("attention_type", ["content_and_conv", "content"])
def test_state_functions_greedy_and_sampled_generation(attention_type):
    """generate(sample=False) emits the oracle's arg-max tokens with its costs and states; sample() draws from a
    device stream, so its costs are checked against the oracle's teacher-forced costs of the drawn tokens."""
    torch = _torch()
    cfg = SO.make_config(attention_type, **dict(SMALL, prior=MEDIAN))
    params = _params(cfg, seed=7, gain=3.0)
    rec = _recognizer(cfg, params)
    B, T, n = 5, 36, 12
    att, attm, att64, attm64, x, m, labels, lm = _encode(rec, cfg, B, T, seed=9)
    got = rec.generate(x, m, n_steps=n, sample=False)
    outs, costs, states = SO.generate_greedy(cfg, params, att64, attm64, n)
    assert np.array_equal(got["outputs"], outs)
    assert elementwise_err(got["costs"], costs) <= TOL["costs"]
    assert elementwise_err(got["states"], states) <= TOL["states"]
    drawn = rec.generate(x, m, n_steps=n, sample=True, seed=4)
    want = SO.cost_matrix(cfg, params, att64, attm64, drawn["outputs"].astype(np.int64))
    assert elementwise_err(drawn["costs"], want) <= TOL["costs"]
    torch.cuda.synchronize()


def _utterances(cfg, seed, lengths=(40, 27, 33, 46)):
    rng = np.random.RandomState(seed)
    return [rng.normal(size=(T, cfg["num_features"])) for T in lengths]


@pytest.mark.parametrize("beam", [1, 10])
@pytest.mark.parametrize("stop_on,char_discount", [("patience", 0.0), ("optimistic_future_cost", 0.1)])
def test_beam_search_matches_oracle(beam, stop_on, char_discount):
    """Every finished hypothesis with its cost, one utterance at a time and in search_many's lock-step."""
    _torch()
    scale = 2.0
    cfg = SO.make_config(max_decoded_length_scale=scale, **dict(SMALL, prior=MEDIAN))
    params = _params(cfg, seed=11, gain=4.0, eos_bias=6.0)
    rec = _recognizer(cfg, params)
    rec.init_beam_search(beam)
    utts = _utterances(cfg, 13)
    many = rec._beam_search.search_many([u.astype(np.float32) for u in utts], cfg["eos_label"],
                                        [int(u.shape[0] / scale) for u in utts], stop_on=stop_on,
                                        char_discount=char_discount, raise_on_failure=False)
    found = 0
    for u, g in zip(utts, many):
        try:
            want = SO.beam_search(cfg, params, u, beam, stop_on=stop_on, char_discount=char_discount)
        except O.CandidateNotFoundError:
            assert g is None
            continue
        found += 1
        one = rec.beam_search({"recordings": u}, stop_on=stop_on, char_discount=char_discount)
        for res in (one, g):        # the attention's cluster size follows the rows in flight: costs may differ in ulps
            if beam == 1:
                assert res[0] == want[0]
                assert elementwise_err(res[1], want[1]) <= 1e-5
            else:
                _same_up_to_near_ties(res, want)
    assert found >= 2


def test_beam_search_with_an_fst_language_model(tmp_path):
    """Shallow fusion touches only the readout: the stacked decoder searches with an LM like the oracle does."""
    _torch()
    V = SMALL["num_phonemes"]
    S, start, arcs = LO.char_ngram(V, seed=7, n_tri=60, dup=6, dead=2)
    path = str(tmp_path / "lm.fst")
    cmap = LO.to_file(path, V, S, start, arcs, seed=2)
    fst = LO.from_tables(package().lm.load(path, cmap, V))
    o = dict(normalize_am_weights=True, normalize_lm_weights=False, normalize_tot_weights=False, am_beta=1.0,
             weight=0.5, no_transition_cost=20.0)
    scale, beam = 2.0, 5
    cfg = SO.make_config(max_decoded_length_scale=scale, **dict(SMALL, prior=MEDIAN))
    params = _params(cfg, seed=11, gain=4.0, eos_bias=6.0)
    rec = _recognizer(cfg, params, lm=dict(o, path=path), cmap=cmap)
    rec.init_beam_search(beam)
    utts = _utterances(cfg, 17)
    got = rec._beam_search.search_many([u.astype(np.float32) for u in utts], cfg["eos_label"],
                                       [int(u.shape[0] / scale) for u in utts], raise_on_failure=False)

    def f_init(att):
        st = SO.initial_states(cfg, params, 1, att)
        s, row = LO.initial(fst, V, o["no_transition_cost"])
        st["lm_sets"] = np.array([s], dtype=object)
        st["lm_add"] = row[None, :]
        return st

    def f_logp(att, m, st):
        wide = SO.wide_params(cfg, params)
        wa, _, _, _ = O.take_glimpses(cfg, wide, att, None, m, st["weights"], st["step"], st["states"])
        return LO.fused_costs(O.readout(cfg, wide, st["states"], wa), st["lm_add"], o)

    def f_next(att, m, st, y):
        nxt = SO.next_state_computer(cfg, params, att, m, OrderedDict((k, v) for k, v in st.items()
                                                                      if not k.startswith("lm_")), y)
        pairs = [LO.next_state(fst, s, yy, V, o["no_transition_cost"]) for s, yy in zip(st["lm_sets"], y)]
        sets = np.empty(len(pairs), dtype=object)
        sets[:] = [p[0] for p in pairs]
        nxt["lm_sets"] = sets
        nxt["lm_add"] = np.stack([p[1] for p in pairs]) if pairs else np.zeros((0, V), np.float32)
        return nxt

    found = 0
    for u, g in zip(utts, got):
        try:
            want = O.beam_search(cfg, params, u, beam, computers=dict(initial=f_init, logprobs=f_logp, next=f_next))
        except O.CandidateNotFoundError:
            assert g is None
            continue
        found += 1
        assert g[0] == want[0]
        assert np.allclose(g[1], want[1], rtol=1e-3, atol=5e-3)
    assert found >= 1


def test_checkpoint_round_trip(tmp_path):
    """save_params writes every stack parameter under its Blocks name; load_params restores them bit for bit."""
    _torch()
    cfg = SO.make_config(**SMALL)
    params = _params(cfg, seed=21)
    rec = _recognizer(cfg, params)
    path = str(tmp_path / "stack.tar")
    rec.save_params(path)
    with tarfile.open(path) as tar:
        keys = set(np.load(tar.extractfile("_parameters")).files)
    assert keys == {k.replace("/", "|") for k in SO.param_shapes(cfg)}
    other = _recognizer(cfg, _params(cfg, seed=22))
    report = other.load_params(path)
    assert report == dict(unknown=[], missing=[])
    got = other.get_parameter_values()
    for k, v in params.items():
        assert np.array_equal(got[k], np.asarray(v, np.float32)), k
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=24, seed=2)
    assert np.array_equal(other.cost(x, m, labels, lm), rec.cost(x, m, labels, lm))
    assert os.path.getsize(path) > 0
