"""The stacked decoder (net.dec_stack: 2) at the widths, row counts, encoded lengths, streams and entry points the
single-layer decoder is tested at, against the float64 stack oracle (tests/stack_oracle.py) element by element.

Both layers run on decoder.cu's dense_kernel: a CTA owns 8 output columns of a block of 64 rows, its 8 warps split
each contraction (E, C, C for the gates, C for the candidate) into slices of ceil(K / 32) float4 groups.  The widths of
test_gpu_widths.py (C = 8, 72 and 200 leave ragged or empty slices) are run here with a stack, both readout settings
(use_states_for_readout=False drops the merge's two state weights, which finalize then leaves unpacked), every readout
activation, one-hot feedback and V = 2 to 128; row counts around the kernel's 64-row blocks (1, 63, 64, 65, 128, 300)
with ragged label masks, whose masked steps must leave both layers' states bit for bit; 72 rows past the longest row
one attention CTA holds (cs 2 at T' = 1289 and 2000, bench.NET's decoder widths); greedy and sampled generation at 100
rows; search_many over the configs[2] shape of bench.py and over long utterances; teacher forcing with an FST language
model; the stream contract on a non-blocking stream; validation_statistics, analyze, pickling and compat's search and
sample.

Every teacher-forced case asserts through SpeechRecognizer.decoder_plan() that the step-wise kernels ran (the persistent
decoder holds one layer).  Bounds are test_gpu_attention_plans.py's TOL (weights 5e-5 relative per element, energies
2e-5 of their scale, weight sums 2e-6, costs 1e-5, states and weighted averages 1e-4, each per element with a floor of
0.1 of the tensor's scale); beams must find the oracle's hypotheses, reordered only between costs within 1e-4, with
search costs within 1e-5 (test_gpu_widths.py).  The oracle decodes the GPU's own encoder output, rounded to float32.

Worst errors measured over this file on an H100 80GB HBM3 (700 W power limit): weights 1.1e-5, energies 1.9e-6 and
weighted averages 2.1e-5 (72 rows at T' = 1289), weight sums 2.0e-7, costs 2.5e-6, states 4.9e-5 (E = C = 512, state
rows of 1024), search costs 6.6e-6, LM-fused costs 3.3e-6 (bound: test_gpu_lm.py's 1e-4), validation_statistics'
cost sum 7.3e-9, entropy 7.6e-8 and penalty 4.4e-5 relative (bound: 1e-5, 5e-5 and the gate, 1e-4).  The file runs
in about a minute there, 35 s of it in the two large searches, most of that the oracle's."""
import pickle
import sys

import numpy as np
import pytest

import lm_oracle as LO
import stack_oracle as SO
import test_gpu_widths as W
import training_loop_oracle as TL
from compat_helpers import COMPAT, write_experiment
from helpers import O, WSJ, check_energies, check_weights, elementwise_err, f32, make_recognizer, package
from test_gpu_attention_plans import TOL, WSUM_TOL, _compare, _set_env
from test_gpu_dec_stack import MEDIAN, SMALL, _params, _recognizer
from test_gpu_lm import FLAGS, lm_file  # noqa: F401  (lm_file: the LM fixture of test_gpu_lm.py)
from test_gpu_stepwise_rows import ARCH as NET, STRESS, _assert_stepwise, _longest_row
from test_gpu_streams import _dev, _equal, _np, _on, stream  # noqa: F401  (stream: default and non-blocking)
from test_gpu_widths import _same_up_to_near_ties

pytestmark = pytest.mark.gpu


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _cuda(a):
    torch = _torch()
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32, device="cuda")


def _width_config(case, **kw):
    """A stack at the widths of test_gpu_widths.CASES[case]."""
    net, prior = W.CASES[case]
    if case.startswith("content"):
        return SO.make_config("content", **dict(W.COMMON, **net, **kw))
    return SO.make_config(prior=prior, **dict(W.COMMON, **net, **kw))


def _errs(got, want, content):
    """The element-wise errors of _compare on numpy arrays, returned instead of asserted."""
    errs = {}
    check_weights(got["weights"], want["weights"], errs)
    if not content:
        check_energies(got["energies"], want["energies"], errs)
    for k in ("costs", "states", "weighted_averages"):
        if k in got:
            errs[k] = elementwise_err(got[k], want[k])
    return errs


def _check(errs, what):
    print("ERRS", what, " ".join("%s=%.2e" % kv for kv in sorted(errs.items())))
    for k, e in errs.items():
        assert e <= (WSUM_TOL if k.endswith("_sum") else TOL[k]), (what, k, e)


def _stack_cost(monkeypatch, cfg, params, inputs, what, rec=None):
    """cost_matrix(return_all) of a stack on given attended arrays against SO.cost_matrix; the step-wise kernels ran.
    Returns the GPU's outputs as numpy arrays and the plan."""
    att, attm, labels, lm = inputs
    rec = rec or make_recognizer(cfg, params)
    assert list(rec.parameter_shapes().items()) == list(SO.param_shapes(cfg).items())
    _set_env(monkeypatch)
    got = rec.cost_matrix(labels, lm, _cuda(att), _cuda(attm), return_all=True)
    plan = rec.decoder_plan()
    print("PLAN", what, {k: plan[k] for k in ("ran", "kernel", "cs", "att_cs")})
    assert rec.launch_status() == (0, 0)
    L, B = labels.shape
    assert tuple(got["states"].shape) == (L, B, 2 * cfg["dim_dec"])
    want = SO.cost_matrix(cfg, params, att, attm, labels, lm, return_all=True)
    got = _compare(got, want, cfg["attention_type"] == "content", what)
    assert not plan["ran"] and plan["kernel"] == "stepwise" and plan["cs"] == 0 and plan["att_cs"] >= 1, plan
    return got, plan


def _encode(rec, x, m):
    """The GPU encoder's output as device tensors and as float64 arrays for the oracle."""
    att, attm = rec.encode(x, m)
    return att, attm, f32(att.cpu().numpy()), attm.cpu().numpy().astype(np.float64)


# ---- 1. widths ---------------------------------------------------------------------------------------------------

WIDTHS = [(c, True) for c in W.CASES] + [("ragged_k", False), ("odd_c", False)]


@pytest.mark.parametrize("case,states_readout", WIDTHS,
                         ids=[c + ("" if s else "-no_states_readout") for c, s in WIDTHS])
def test_cost_matrix_at_every_width(case, states_readout, monkeypatch):
    """Costs, weights, energies, both layers' states [L, B, 2C] and the glimpses at C = 8 (every slice of layer 1's
    contractions empty but the first), 72 and 200 (a ragged last slice), 384, 512; without the states in the readout
    (Maxout(3) and Tanh), the merge weights are not in the table and the stack's packed copy of them is not read."""
    _torch()
    cfg = _width_config(case, use_states_for_readout=states_readout)
    params = _params(cfg, seed=3 + len(case))
    if not states_readout:
        assert not any("readout/merge/transform_states" in k for k in params)
    inputs = W._inputs(cfg, 5, 30, 7, seed=11 + len(case))
    _stack_cost(monkeypatch, cfg, params, inputs, "%s%s" % (case, "" if states_readout else " no states readout"))


@pytest.mark.parametrize("case", ["odd_c", "e512_c128"])
def test_greedy_generate_at_width(case, monkeypatch):
    """generate(sample=False) on 3 rows: the oracle's arg-max tokens, their costs and both layers' states."""
    _torch()
    cfg = _width_config(case)
    params = _params(cfg, seed=31, gain=3.0)
    rec = make_recognizer(cfg, params)
    _set_env(monkeypatch)
    x, m, _, _ = O.synthetic_batch(cfg, B=3, T=30, seed=32)
    _, _, att64, attm64 = _encode(rec, x, m)
    n = 6
    got = rec.generate(x, m, n_steps=n, sample=False)
    outs, costs, states = SO.generate_greedy(cfg, params, att64, attm64, n)
    assert np.array_equal(got["outputs"], outs)
    _check(dict(costs=elementwise_err(got["costs"], costs), states=elementwise_err(got["states"], states)),
           "greedy %s" % case)
    _assert_stepwise(rec.decoder_plan(), 3, att64.shape[0])


@pytest.mark.parametrize("stop_on,char_discount", [("patience", 0.0), ("optimistic_future_cost", 0.1)])
def test_search_many_ragged_k(stop_on, char_discount):
    """search_many at beam 5 on the C = 72 stack: every finished hypothesis of the oracle with its cost."""
    _torch()
    scale = 2.0
    cfg = _width_config("ragged_k", max_decoded_length_scale=scale)
    params = _params(cfg, seed=41, gain=4.0, eos_bias=4.0)
    rng = np.random.RandomState(42)
    utts = [f32(rng.normal(size=(T, cfg["num_features"]))) for T in (36, 25, 30)]
    rec = make_recognizer(cfg, params)
    got = W._search(rec, cfg, utts, 5, scale, stop_on=stop_on, char_discount=char_discount)
    n_hyp = 0
    for u, g in zip(utts, got):
        try:
            want = SO.beam_search(cfg, params, u, 5, stop_on=stop_on, char_discount=char_discount)
        except O.CandidateNotFoundError:
            assert g is None
            continue
        assert g is not None
        n_hyp += _same_up_to_near_ties(g, want)
    assert n_hyp >= 2


# ---- 2. rows around the stack kernel's 64-row blocks --------------------------------------------------------------

@pytest.mark.parametrize("B", [1, 63, 64, 65, 128, 300])
def test_rows_around_the_row_blocks(B, monkeypatch):
    """A full or partial last block of 64 rows; label lengths from 1 to L, so that masked trailing steps leave both
    layers' states exactly as they were."""
    _torch()
    cfg = SO.make_config(**dict(SMALL, prior=MEDIAN))
    params = _params(cfg, seed=5)
    L = 9
    att, attm, labels, _ = W._inputs(cfg, B, 32, L, seed=B)
    lens = np.random.RandomState(B + 1).randint(1, L + 1, size=B)
    lens[0] = L
    lm = (np.arange(L)[:, None] < lens[None, :]).astype(np.float64)
    got, _ = _stack_cost(monkeypatch, cfg, params, (att, attm, labels, lm), "rows B=%d" % B)
    # states[i] is the state before step i: after the last unmasked step n - 1 it no longer changes
    for b, n in enumerate(lens):
        for i in range(n + 1, L):
            assert np.array_equal(got["states"][i, b], got["states"][n, b]), (b, n, i)


@pytest.mark.parametrize("sample", [False, True], ids=["greedy", "sampled"])
def test_generate_at_100_rows(sample, monkeypatch):
    """generate on 100 rows: greedy against the oracle's arg-max, sampled against the oracle's teacher-forced costs of
    the drawn tokens."""
    _torch()
    cfg = SO.make_config(**dict(SMALL, prior=MEDIAN))
    params = _params(cfg, seed=7, gain=3.0)
    rec = make_recognizer(cfg, params)
    _set_env(monkeypatch)
    B, n = 100, 8
    x, m, _, _ = O.synthetic_batch(cfg, B=B, T=36, seed=9)
    _, _, att64, attm64 = _encode(rec, x, m)
    got = rec.generate(x, m, n_steps=n, sample=sample, seed=4)
    if sample:
        want = SO.cost_matrix(cfg, params, att64, attm64, got["outputs"].astype(np.int64))
        errs = dict(costs=elementwise_err(got["costs"], want))
    else:
        outs, costs, states = SO.generate_greedy(cfg, params, att64, attm64, n)
        assert np.array_equal(got["outputs"], outs)
        errs = dict(costs=elementwise_err(got["costs"], costs), states=elementwise_err(got["states"], states))
    _check(errs, "generate 100 rows sample=%s" % sample)
    _assert_stepwise(rec.decoder_plan(), B, att64.shape[0])


# ---- 3. long encoded lengths ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("where", ["cs1_limit_plus_1", "t2000"])
def test_long_rows(where, monkeypatch):
    """72 rows at bench.NET's decoder widths (E = M = 512, C = 256) one position past the longest row one attention CTA
    holds, and at T' = 2000: clusters of 2 under the stress prior."""
    _torch()
    Tp = _longest_row(1) + 1 if where == "cs1_limit_plus_1" else 2000
    cfg = SO.make_config(prior=STRESS, **NET)
    params = _params(cfg, seed=5)
    inputs = W._inputs(cfg, 72, Tp, 4, seed=Tp)
    _, plan = _stack_cost(monkeypatch, cfg, params, inputs, "long T'=%d" % Tp)
    _assert_stepwise(plan, 72, Tp)
    assert plan["att_cs"] == 2, plan


# ---- 4. search at scale ---------------------------------------------------------------------------------------------

def _search_vs_oracle(cfg, params, utts, beam, scale, compare):
    """search_many over all `utts`; the utterances `compare` against SO.beam_search one by one."""
    rec = make_recognizer(cfg, params)
    rec.init_beam_search(beam)
    got = rec._beam_search.search_many([u.astype(np.float32) for u in utts], cfg["eos_label"],
                                       [int(u.shape[0] / scale) for u in utts], raise_on_failure=False)
    n_found = n_hyp = 0
    for i in compare:
        try:
            want = SO.beam_search(cfg, params, utts[i], beam)
        except O.CandidateNotFoundError:
            assert got[i] is None
            continue
        assert got[i] is not None and got[i][0][0] == want[0][0], (i, got[i], want)
        n_hyp += _same_up_to_near_ties(got[i], want)
        n_found += 1
    print("utterances with a result:", n_found, "finished hypotheses compared:", n_hyp)
    assert n_found >= 1 and n_hyp > n_found
    return rec.decoder_plan()


def test_search_many_wsj_shape():
    """bench.py's configs[2] shape with a stack: 32 utterances of 480-800 frames (T' <= 200) at beam 10, up to 320
    rows in lock-step (gather_rows moves state rows of 2C), eight of them compared with the oracle."""
    _torch()
    scale = 8.0
    cfg = SO.make_config(max_decoded_length_scale=scale, **WSJ)
    params = _params(cfg, seed=91, gain=4.0, eos_bias=2.0)
    rng = np.random.RandomState(92)
    lens = rng.randint(480, 801, size=32)
    lens[0] = 800
    utts = [f32(rng.normal(size=(T, cfg["num_features"]))) for T in lens]
    plan = _search_vs_oracle(cfg, params, utts, 10, scale, compare=(0, 4, 9, 13, 18, 22, 27, 31))
    assert not plan["ran"] and plan["att_cs"] >= 1, plan


def test_search_many_long_utterances():
    """8 utterances of 1300-1500 frames at beam 10 under the stress prior: 8 rows at cs 8, then up to 80 rows that one
    CTA per row cannot hold; two of them compared with the oracle."""
    _torch()
    scale = 100.0
    cfg = SO.make_config(prior=STRESS, max_decoded_length_scale=scale, **NET)
    params = _params(cfg, seed=81, gain=4.0, eos_bias=2.0)
    rng = np.random.RandomState(82)
    utts = [f32(rng.normal(size=(T, cfg["num_features"]))) for T in rng.randint(1300, 1501, size=8)]
    assert min(u.shape[0] for u in utts) > _longest_row(1)
    plan = _search_vs_oracle(cfg, params, utts, 10, scale, compare=(0, 5))
    assert plan["att_cs"] >= 2, plan


# ---- 5. teacher forcing with a language model -----------------------------------------------------------------------

@pytest.mark.parametrize("attention", ["content_and_conv", "content"])
def test_fused_cost_matrix(lm_file, attention):
    """cost_matrix with the FST LM attached against the oracle composition of test_gpu_lm.py over the stack oracle:
    the fused readout of SO's states and glimpses, for every normalisation setting, two AM weights and two LM weights."""
    _torch()
    path, cmap, fst = lm_file
    cfg = SO.make_config(attention, **dict(SMALL, prior=MEDIAN))
    V = cfg["num_phonemes"]
    params = _params(cfg, seed=4)
    rec = _recognizer(cfg, params, lm=dict(path=path, no_transition_cost=20.0), cmap=cmap)
    x, m, labels, lmask = O.synthetic_batch(cfg, B=3, T=40, seed=5)
    att, attm, att64, attm64 = _encode(rec, x, m)
    r = SO.cost_matrix(cfg, params, att64, attm64, labels, lmask, return_all=True)
    logits = O.readout(cfg, SO.wide_params(cfg, params), r["states"], r["weighted_averages"])
    lib, h = package()._lib.load(), rec._require_ready()
    n, worst = 0, 0.0
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
                    got = rec.cost_matrix(labels, lmask, att, attm).cpu().numpy().astype(np.float64)
                    want = np.take_along_axis(LO.fused_costs(logits, add, o), labels[..., None], axis=-1)[..., 0] * lmask
                    assert np.allclose(got, want, rtol=1e-4, atol=1e-4), (o, np.abs(got - want).max())
                    worst = max(worst, elementwise_err(got, want))
                    n += 1
    print("settings compared:", n, "worst fused cost error %.2e" % worst)
    plan = rec.decoder_plan()
    assert not plan["ran"] and plan["kernel"] == "stepwise", plan


# ---- 6. the stream contract -----------------------------------------------------------------------------------------

def _stack_calls(rec, s, cfg, batch, utts, delay):
    """cost_matrix(return_all), beam_search_many at beam 5 and greedy generate on s, each behind a queued spin."""
    x, m, labels, lm = batch
    xd, md, yd, ymd = _dev(s, x, m, labels, lm)
    att, attm = _on(s, rec.encode, xd, md, delay=False)
    out = _on(s, rec.cost_matrix, yd, ymd, att, attm, return_all=True, delay=delay)
    rec.init_beam_search(5)
    found = _on(s, rec.beam_search_many, [{"recordings": u} for u in utts], delay=delay)
    gen = _on(s, rec.generate, x, m, n_steps=8, sample=False, delay=delay)
    s.synchronize()
    return dict(att=att.cpu().numpy(), attm=attm.cpu().numpy(), all=_np(out), search=found, gen=gen)


def test_stack_is_ordered_on_the_stream(stream):
    """The stacked step's copies and workspace buffers follow the caller's stream: a warm handle's answers behind a
    queued spin are the serial default-stream answers bit for bit, and the cost matrix is the oracle's."""
    torch = _torch()
    cfg = SO.make_config(max_decoded_length_scale=3.0, **dict(SMALL, prior=MEDIAN))
    params = _params(cfg, seed=11, gain=4.0, eos_bias=6.0)
    batch = O.synthetic_batch(cfg, B=6, T=48, seed=21)
    rng = np.random.RandomState(5)
    utts = [rng.normal(size=(T, cfg["num_features"])).astype(np.float32) for T in (64, 37, 52, 45)]
    serial = _stack_calls(make_recognizer(cfg, params), torch.cuda.default_stream(), cfg, batch, utts, delay=False)
    rec = make_recognizer(cfg, params)
    warm = _stack_calls(rec, stream, cfg, batch, utts, delay=False)
    got = _stack_calls(rec, stream, cfg, batch, utts, delay=True)
    for k in ("att", "all", "search", "gen"):
        assert _equal(warm[k], serial[k]) and _equal(got[k], serial[k]), k
    assert any(g is not None for g in got["search"])
    want = SO.cost_matrix(cfg, params, f32(got["att"]), got["attm"].astype(np.float64), batch[2], batch[3],
                          return_all=True)
    _check(_errs({k: v.astype(np.float64) for k, v in got["all"].items()}, want, False),
           "stream %s" % ("default" if stream.cuda_stream == 0 else "side"))


# ---- 7. entry points ------------------------------------------------------------------------------------------------

def test_validation_statistics_and_analyze():
    """validation_statistics: the summed costs, the alignment entropy and penalty of the oracle's weights;
    analyze: one utterance's costs, weights and energies."""
    _torch()
    cfg = SO.make_config(**dict(SMALL, prior=MEDIAN))
    params = _params(cfg, seed=3)
    rec = make_recognizer(cfg, params)
    x, m, labels, lm = O.synthetic_batch(cfg, B=5, T=48, seed=11)
    s = rec.validation_statistics(x, m, labels, lm)
    _, _, att64, attm64 = _encode(rec, x, m)
    want = SO.cost_matrix(cfg, params, att64, attm64, labels, lm, return_all=True)
    ent, pen = TL.alignment_stats(want["weights"], lm)
    errs = dict(cost=abs(s["cost"] - want["costs"].sum()) / abs(want["costs"].sum()),
                entropy=abs(s["weights_entropy"] - ent) / abs(ent), penalty=abs(s["weights_penalty"] - pen) / abs(pen))
    print("ERRS validation_statistics", " ".join("%s=%.2e" % kv for kv in sorted(errs.items())))
    assert errs["cost"] <= TOL["costs"] and errs["entropy"] <= TOL["weights"] and errs["penalty"] <= 1e-4, errs
    assert s["num_labels"] == float(lm.sum()) and s["batch_size"] == 5
    # analyze: the reference's one-utterance cost graph, mask of ones, no label mask
    T, n = int(m[:, 1].sum()), int(lm[:, 1].sum())
    u, y = x[:T, 1], labels[:n, 1]
    costs, weights, energies = rec.analyze({"recordings": u}, y)
    _, _, att64, attm64 = _encode(rec, u[:, None, :], np.ones((T, 1)))
    want = SO.cost_matrix(cfg, params, att64, attm64, y[:, None], None, return_all=True)
    errs = {}
    check_weights(weights, want["weights"][:, 0], errs)
    check_energies(energies, want["energies"][:, 0], errs)
    errs["costs"] = elementwise_err(costs, want["costs"][:, 0])
    _check(errs, "analyze")
    _assert_stepwise(rec.decoder_plan(), 1, att64.shape[0])


def test_pickle_round_trip():
    """A pickled stack carries its configuration and parameters: the unpickled recognizer's costs are bit-identical."""
    _torch()
    cfg = SO.make_config(**dict(SMALL, prior=MEDIAN))
    rec = make_recognizer(cfg, _params(cfg, seed=21))
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=24, seed=2)
    before = rec.cost(x, m, labels, lm)
    back = pickle.loads(pickle.dumps(rec))
    assert back.dim_state == 2 * cfg["dim_dec"] and back._make_config().dec_stack == 2
    assert np.array_equal(back.cost(x, m, labels, lm), before)


def test_compat_search_and_sample(tmp_path, capsys):
    """compat's search and sample on a net.dec_stack=2 experiment from a checkpoint of stack-oracle parameters: the
    report lines, and the tokens of recognizer.beam_search and recognizer.sample on the same utterances."""
    _torch()
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as LC
    import lvsr.main as LM
    exp = write_experiment(tmp_path)
    config = LC.Configuration(exp["base"], "$LVSR/lvsr/configs/schema.yaml", [("net.dec_stack", "2")])
    data = LM.Data(**config["data"])
    net = config["net"]
    cfg = SO.make_config(num_features=data.num_features, dims_bidir=net["dims_bidir"], subsample=net["subsample"],
                         dim_dec=net["dim_dec"], conv_n=net["conv_n"], conv_num_filters=net["conv_num_filters"],
                         num_phonemes=data.num_labels, eos_label=data.eos_label, post_merge_dims=net["post_merge_dims"],
                         maxout_pieces=2, max_decoded_length_scale=net["max_decoded_length_scale"])
    model = LM.create_model(config, data)
    assert list(model.parameter_shapes().items()) == list(SO.param_shapes(cfg).items())
    params = _params(cfg, seed=23, gain=4.0, eos_bias=6.0)
    model.set_parameter_values(params)
    path = str(tmp_path / "stack.tar")
    model.save_params(path)
    decoded = str(tmp_path / "decoded.txt")
    capsys.readouterr()
    LM.search(config, None, path, "valid", None, None, decoded, False, 1)
    out = capsys.readouterr().out
    for line in ("Utterance 2", "Groundtruth cost:", "Beam search cost:", "Recognized:", "Average CER:"):
        assert line in out, line
    sc = config["monitoring"]["search"]
    kw = {k: v for k, v in dict(char_discount=sc.get("char_discount"), round_to_inf=sc.get("round_to_inf"),
                                 stop_on=sc.get("stop_on")).items() if v}
    model.init_beam_search(sc["beam_size"])
    dataset = data.get_dataset("valid")
    want, samples, found = [], [], 0
    for example in data.examples("valid", shuffle=False, seed=1):
        uttid = example.pop("uttids", None)
        example.pop("labels")
        inputs = {k: v for k, v in example.items() if k in model.inputs}
        try:
            outputs = model.beam_search(inputs, **kw)[0]
            found += 1
        except package().CandidateNotFoundError:
            outputs = [[]]
        want.append("{} {}".format(uttid, " ".join(dataset.decode(outputs[0]))))
        samples.append(dataset.pretty_print(model.sample(inputs)[:, 0], example))
    with open(decoded) as f:
        assert f.read().splitlines() == want
    assert found >= 1
    LM.sample(config, None, path, "valid")
    out = capsys.readouterr().out
    for number, text in enumerate(samples):
        assert "Utterance %d\n%s\n" % (number, text) in out, number
