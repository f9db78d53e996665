"""The decoder, readout, search and training step at decoder, matcher, feedback and readout widths away from the 128 /
256 of the other tests, compared with the float64 oracle element by element.

lvsr_model_create takes any dim_dec and post_merge_dim that is a multiple of 8, any dim_output_embedding that is a
multiple of 4, dim_matcher 128, 256 or 512, any Maxout piece count that divides post_merge_dim and 1 to 128 symbols.
The kernels cut their contractions by these widths: dense_kernel and skinny_kernel into per-warp float4 slices (C = 8,
72 and 200 leave ragged or empty slices), readout_kernel / readout_bwd_kernel into Maxout groups of 3 or 4 pieces, the
persistent decoder into KPER = 16 or 24 k-values per lane (C = 512).  Each case below names the decoder it runs (the
persistent one needs E + C and C to be one of its product shapes, dec_scan.cu kper_ok), asserts through
SpeechRecognizer.decoder_plan() that this decoder ran, and compares with O.cost_matrix (content_oracle for content
attention) run on the float32-rounded inputs and parameters:

  * weights: relative error per element wherever the oracle weight is >= 1e-30, exactly 0 where the oracle's is 0;
  * energies: absolute error per element over the tensor's largest magnitude, exactly 0 outside the window;
  * costs, states, weighted averages, log-probabilities: |got - want| <= tol * (|want| + 0.1 * max|want|).

The bounds in TOL sit 4-10x above the largest error measured for each quantity over every case of this file on an
H100 80GB HBM3 (400 W power limit), except where that would be looser than 1e-4, the project's gate.  Search results are
compared token for token; the training step through helpers.check_grads (worst gradient error measured: 2.0e-5 of the
parameter's largest entry).  The file runs in about 20 s on that GPU.

Which (E, C) pairs the persistent decoder takes: kper_ok needs E + C and C to be multiples of 128 with 4, 8, 12, 16 or 24
k-values per lane, so with E = 256 it runs at C = 128, 256 and 512 (E + C = 768: KPER = 24 in the gate product, 16 in the
candidate and query products), with E = 512 at C = 256 only; (256, 384), (512, 128) and (512, 512) give E + C = 640 or
1024 and always run on the step-wise kernels, as does any C that is not a multiple of 128.  Mutants that each change
only values (dense_kernel and skinny_kernel slices of K / 32 and K / 64 float4 groups, Maxout pieces indexed j * 2 + p in
both readout kernels, the persistent decoder's candidate and query weights staged as zeros from row 256 on) each fail
tests here; the GPU suite without this file passes with all four.
"""
import math

import numpy as np
import pytest

import content_oracle as CO
from helpers import O, PYRAMID, check_energies, check_grads, check_weights, elementwise_err, f32, make_recognizer
from helpers import train_like_the_oracle
from oracle import lvsr_oracle_grad as G

pytestmark = pytest.mark.gpu

# per-quantity bounds; the largest error measured over every case of this file is in the comment.  States and weighted
# averages stay at the gate, 2.6x and 3.9x above their measured errors.
TOL = dict(weights=1e-4,             # 1.8e-5 relative, per element (E = 512, C = 512)
           energies=3e-5,            # 5.6e-6 of the tensor's largest magnitude
           costs=3e-5,               # 5.3e-6
           logprobs=4e-6,            # 6.9e-7
           states=1e-4,              # 3.9e-5
           weighted_averages=1e-4,   # 2.6e-5
           search_costs=1e-5)        # 1.6e-6: cumulative costs of the finished hypotheses
WSUM_TOL = 1e-6                      # 1.6e-7

MEDIAN = dict(type="window_around_median", before=5, after=7)
MEAN = dict(type="window_around_mean", before=6, after=6)

E256 = dict(dims_bidir=[128], subsample=[1])               # BiGRU(128): E = 256
COMMON = dict(num_features=40, conv_n=8, conv_num_filters=10)

# name -> (network, prior); dim_output_embedding is the feedback width (dim_dec when absent)
CASES = {
    "tiny": (dict(E256, dim_dec=8, dim_matcher=128, dim_output_embedding=4, post_merge_dims=[8], maxout_pieces=2,
                  num_phonemes=2), MEDIAN),
    "ragged_k": (dict(E256, dim_dec=72, dim_matcher=256, dim_output_embedding=12, post_merge_dims=[24],
                      maxout_pieces=3, num_phonemes=33), MEAN),
    "odd_c": (dict(E256, dim_dec=200, dim_matcher=128, dim_output_embedding=100, post_merge_dims=[200],
                   post_merge_activation="tanh", num_phonemes=97), MEDIAN),
    "c384": (dict(E256, dim_dec=384, dim_matcher=512, dim_output_embedding=260, post_merge_dims=[264],
                  maxout_pieces=3, num_phonemes=128), MEAN),
    "c512": (dict(E256, dim_dec=512, dim_matcher=256, post_merge_dims=[512], maxout_pieces=4, num_phonemes=127),
             MEDIAN),
    "c512_onehot": (dict(E256, dim_dec=512, dim_matcher=512, embed_outputs=False, post_merge_dims=[256],
                         maxout_pieces=2, num_phonemes=31), MEAN),
    "e512_c128": (dict(dims_bidir=[256, 256], subsample=[1, 2], dim_dec=128, dim_matcher=128, post_merge_dims=[128],
                       post_merge_activation="relu", num_phonemes=64), MEDIAN),
    "e512_c512": (dict(dims_bidir=[256, 256], subsample=[1, 1], dim_dec=512, dim_matcher=512, post_merge_dims=[512],
                       post_merge_activation="identity", num_phonemes=32), MEAN),
    "content_c512": (dict(E256, dim_dec=512, dim_matcher=256, post_merge_dims=[256], maxout_pieces=2, num_phonemes=32),
                     None),
}


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _config(case, **kw):
    net, prior = CASES[case]
    if case.startswith("content"):
        return CO.make_config(**dict(COMMON, **net, **kw))
    return O.make_config(prior=prior, **dict(COMMON, **net, **kw))


def _params(cfg, seed):
    content = cfg["attention_type"] == "content"
    return {k: f32(v) for k, v in (CO if content else O).init_params(cfg, seed=seed, scale=10.0).items()}


def _inputs(cfg, B, Tp, L, seed):
    """attended [T',B,E] in (-1, 1) like a GRU output, ragged lengths (one row full), labels and a label mask with
    trailing zeros."""
    rng = np.random.RandomState(seed)
    lens = rng.randint(int(math.ceil(0.6 * Tp)), Tp + 1, size=B)
    lens[rng.randint(B)] = Tp
    att = f32(rng.uniform(-1, 1, size=(Tp, B, O.dim_encoded(cfg))))
    attm = (np.arange(Tp)[:, None] < lens[None, :]).astype(np.float64)
    labels = rng.randint(0, max(1, cfg["num_phonemes"] - 1), size=(L, B)).astype(np.int64)
    lm = (np.arange(L)[:, None] < rng.randint(max(1, L - 3), L + 1, size=B)[None, :]).astype(np.float64)
    return att, attm, labels, lm


def _set_env(monkeypatch, stepwise=False):
    for k in ("LVSR_DEC_CS", "LVSR_DEC_LAYOUT", "LVSR_DEC_HANDLER", "LVSR_ATT_CS", "LVSR_NO_DEC_SCAN"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("LVSR_DEC_CHECK", "1")       # launch status 0 and no sentinel word left, or the call fails
    if stepwise:
        monkeypatch.setenv("LVSR_NO_DEC_SCAN", "1")


def _check(errs, what):
    print("ERRS", what, " ".join("%s=%.2e" % kv for kv in sorted(errs.items())))
    for k, e in errs.items():
        bound = WSUM_TOL if k.endswith("_sum") else TOL[k]
        assert e <= bound, (what, k, e, bound)


def _cost_vs_oracle(monkeypatch, cfg, params, inputs, want, what, stepwise=False):
    """One cost_matrix call compared with the oracle's outputs `want`; returns the decoder plan it ran."""
    torch = _torch()
    att, attm, labels, lm = inputs
    rec = make_recognizer(cfg, params)
    _set_env(monkeypatch, stepwise)
    got = rec.cost_matrix(labels, lm, torch.as_tensor(att, dtype=torch.float32, device="cuda"),
                          torch.as_tensor(attm, dtype=torch.float32, device="cuda"), return_all=True)
    plan = rec.decoder_plan()
    print("PLAN", what, plan)
    assert rec.launch_status() == (0, 0)
    got = {k: v.double().cpu().numpy() for k, v in got.items()}
    errs = {}
    check_weights(got["weights"], want["weights"], errs)
    if cfg["attention_type"] == "content":
        assert not got["energies"].any(), what
    else:
        check_energies(got["energies"], want["energies"], errs)
    for k in ("costs", "states", "weighted_averages"):
        errs[k] = elementwise_err(got[k], want[k])
    _check(errs, what)
    return plan


# ---- forward: every output of the teacher-forced decoder ----------------------------------------------------------

# (case, B, T', decoder): "stepwise" or (kernel, layout, cs); cs None = the planner's choice
FORWARD = [
    ("tiny", 5, 30, "stepwise"),
    ("ragged_k", 5, 30, "stepwise"),
    ("odd_c", 5, 30, "stepwise"),
    ("c384", 5, 30, "stepwise"),                        # E + C = 640: 20 k-values per lane, not a dec_scan shape
    ("c512", 6, 24, ("dec_scan", "global", 1)),         # ceil(24 / 2) < 16: cs 1
    ("c512", 16, 67, ("dec_scan", "islands", 4)),       # cs 1 and 2 leave tiles of 32 and 16 units (> 8 x 3 columns)
    ("c512_onehot", 6, 30, ("dec_scan", "global", None)),
    ("e512_c128", 5, 30, "stepwise"),                   # E + C = 640
    ("e512_c512", 5, 30, "stepwise"),                   # E + C = 1024: 32 k-values per lane
    ("content_c512", 6, 30, ("dec_content", "global", None)),
]


@pytest.mark.parametrize("case,B,Tp,decoder", FORWARD, ids=["%s-B%d" % (c[0], c[1]) for c in FORWARD])
def test_cost_matrix_matches_oracle(case, B, Tp, decoder, monkeypatch):
    cfg = _config(case)
    params = _params(cfg, seed=B + len(case))
    inputs = _inputs(cfg, B, Tp, 7, seed=B * 3 + len(case))
    want = (CO if case.startswith("content") else O).cost_matrix(cfg, params, *inputs, return_all=True)
    plan = _cost_vs_oracle(monkeypatch, cfg, params, inputs, want, "%s B=%d" % (case, B))
    if decoder == "stepwise":
        assert not plan["ran"] and plan["kernel"] == "stepwise" and plan["cs"] == 0, plan
        assert plan["att_cs"] >= 1, plan
        return
    kernel, layout, cs = decoder
    assert plan["ran"] and plan["kernel"] == kernel, plan
    if layout == "islands":
        assert plan["nisl"] == -(-B // 16) and plan["nrg"] == 1 and plan["grid"] == B * plan["cs"], plan
    else:
        assert plan["nisl"] == 0 and plan["nrg"] == -(-B // 16), plan
    if cs is not None:
        assert plan["cs"] == cs, plan
    # 512 units: at most 8 per CTA in each of the gate / candidate / query tiles
    assert plan["nc2"] == 8 and plan["nc1"] == 24, plan
    # the step-wise kernels on the same inputs
    plan = _cost_vs_oracle(monkeypatch, cfg, params, inputs, want, "%s B=%d step-wise" % (case, B), stepwise=True)
    assert not plan["ran"] and plan["kernel"] == "stepwise", plan


# ---- greedy steps through the search's state functions ------------------------------------------------------------

@pytest.mark.parametrize("case", ["odd_c", "c512", "e512_c128"])
def test_greedy_steps_match_oracle(case, monkeypatch):
    """Six steps of logprobs_computer / next_state_computer on 3 rows of different lengths."""
    torch = _torch()
    cfg = _config(case)
    params = _params(cfg, seed=31)
    Tp, R = 30, 3
    att, attm, _, _ = _inputs(cfg, R, Tp, 1, seed=32)
    attm = (np.arange(Tp)[:, None] < np.array([Tp, Tp - 4, Tp - 9])[None, :]).astype(np.float64)
    rec = make_recognizer(cfg, params)
    _set_env(monkeypatch)
    ctx = dict(attended=torch.as_tensor(att, dtype=torch.float32, device="cuda"),
               attended_mask=torch.as_tensor(attm, dtype=torch.float32, device="cuda"))
    st_o = O.initial_states(cfg, params, R, att)
    st_g = rec._initial_states(Tp, R)
    for step in range(6):
        lp_o = O.logprobs_computer(cfg, params, att, attm, st_o)
        lp_g = rec._logprobs(ctx, st_g).double().cpu().numpy()
        errs = dict(logprobs=elementwise_err(lp_g, lp_o))
        y = lp_o.argmin(axis=1)
        st_o = O.next_state_computer(cfg, params, att, attm, st_o, y)
        st_g = rec._next_states(ctx, st_g, y)
        g = {k: v.double().cpu().numpy() for k, v in st_g.items()}
        check_weights(g["weights"], st_o["weights"], errs)
        check_energies(g["energies"], st_o["energies"], errs)
        errs["states"] = elementwise_err(g["states"], st_o["states"])
        errs["weighted_averages"] = elementwise_err(g["weighted_averages"], st_o["weighted_averages"])
        _check(errs, "%s step %d" % (case, step))
        assert np.array_equal(g["step"], st_o["step"])


# ---- beam search ------------------------------------------------------------------------------------------------

def _peaky(cfg, seed, gain=10.0, eos_bias=1.0):
    """Parameters whose readout is sharp enough that hypotheses finish within the length limit."""
    params = _params(cfg, seed)
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.W"] = f32(
        params["/recognizer/generator/readout/post_merge/mlp/linear_0.W"] * gain)
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.b"][cfg["eos_label"]] = eos_bias
    return params


def _search(rec, cfg, utts, beam, scale, **kw):
    rec.init_beam_search(beam)
    return rec._beam_search.search_many([u.astype(np.float32) for u in utts], cfg["eos_label"],
                                        [int(u.shape[0] / scale) for u in utts], raise_on_failure=False, **kw)


# (case, beam, readout gain, eos bias): V = 2 only at beam 1, since the reference's _smallest takes `beam` of the
# width x V candidates, which must outnumber it; gain and bias chosen so that every utterance finishes hypotheses of
# several lengths
SEARCH = [("tiny", 1, 10.0, 1.0), ("odd_c", 5, 4.0, 8.0), ("c512", 5, 4.0, 8.0), ("e512_c128", 5, 4.0, 4.0)]


@pytest.mark.parametrize("case,beam,gain,eos_bias", SEARCH, ids=[c[0] for c in SEARCH])
@pytest.mark.parametrize("stop_on,char_discount", [("patience", 0.0), ("optimistic_future_cost", 0.1)])
def test_search_many_matches_oracle(case, beam, gain, eos_bias, stop_on, char_discount):
    _torch()
    scale = 2.0
    cfg = _config(case, max_decoded_length_scale=scale)
    params = _peaky(cfg, 41, gain=gain, eos_bias=eos_bias)
    rng = np.random.RandomState(42)
    utts = [f32(rng.normal(size=(T, cfg["num_features"]))) for T in (36, 25, 30)]
    rec = make_recognizer(cfg, params)
    got = _search(rec, cfg, utts, beam, scale, stop_on=stop_on, char_discount=char_discount)
    n_hyp, err = 0, 0.0
    for u, g in zip(utts, got):
        try:
            want = O.beam_search(cfg, params, u, beam, stop_on=stop_on, char_discount=char_discount)
        except O.CandidateNotFoundError:
            assert g is None
            continue
        assert g is not None and g[0] == want[0], (g, want)
        err = max(err, elementwise_err(g[1], want[1]))
        n_hyp += len(want[0])
    _check(dict(search_costs=err), "search %s beam %d %s" % (case, beam, stop_on))
    assert n_hyp >= 1


def _same_up_to_near_ties(got, want):
    """The same finished hypotheses with the same costs; two of them may change places in the ranking only where their
    costs are within 1e-4 relative (float32 against float64 ranking)."""
    g_out, g_cost = got
    w_out, w_cost = want
    assert sorted(map(tuple, g_out)) == sorted(map(tuple, w_out))
    w_rank = {tuple(o): i for i, o in enumerate(w_out)}
    ranks = [w_rank[tuple(o)] for o in g_out]
    _check(dict(search_costs=elementwise_err(g_cost, np.asarray(w_cost)[ranks])), "wide beam")
    for i in range(len(ranks)):
        for j in range(i + 1, len(ranks)):
            if ranks[i] > ranks[j]:
                a, b = w_cost[ranks[i]], w_cost[ranks[j]]
                assert abs(a - b) <= 1e-4 * max(abs(a), abs(b)), (i, j, a, b)
    return len(g_out)


@pytest.mark.parametrize("beam,V", [(200, 32), (100, 128)])
def test_wide_beams_match_oracle(beam, V):
    """Beam 200 at V = 32 (the reference's WSJ accuracy setting) and beam 100 at V = 128, whose 100 x 128 candidate
    table (51 KB) needs segment_topk's opt-in to more than 48 KB of shared memory.  Beam 512 at V = 128 (256 KB) is
    refused with an error, and the recognizer searches as before afterwards."""
    _torch()
    scale = 3.0
    cfg = O.make_config(max_decoded_length_scale=scale, **dict(PYRAMID, num_phonemes=V))
    params = _peaky(cfg, 51, gain=1.0, eos_bias=4.0)
    rng = np.random.RandomState(52)
    utts = [f32(rng.normal(size=(T, cfg["num_features"]))) for T in (44, 33)]
    rec = make_recognizer(cfg, params)
    got = _search(rec, cfg, utts, beam, scale, as_arrays=False)
    n_hyp = 0
    for u, g in zip(utts, got):
        want = O.beam_search(cfg, params, u, beam)
        assert g is not None
        assert g[0][0] == want[0][0]                       # the best hypothesis
        n_hyp += _same_up_to_near_ties(g, want)
    print("finished hypotheses compared:", n_hyp)
    assert n_hyp > beam // 2
    if V == 128:
        before = _search(rec, cfg, utts, beam, scale, as_arrays=True)
        with pytest.raises(RuntimeError, match="does not fit the selection kernel"):
            _search(rec, cfg, utts, 512, scale)
        after = _search(rec, cfg, utts, beam, scale, as_arrays=True)
        for a, b in zip(before, after):
            assert all(np.array_equal(x, y) for x, y in zip(a, b))


# ---- training ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", ["ragged_k", "odd_c", "c384", "c512", "e512_c128", "e512_c512"])
def test_gradients_match_oracle(case):
    """skinny_kernel with ragged K slices, readout_bwd_kernel with Maxout(3) / (4), Tanh, Rectifier and Identity at
    new hidden widths, att_bwd_kernel at M = 128, the feedback-gradient GEMMs at new feedback widths."""
    _torch()
    cfg = _config(case)
    params = O.init_params(cfg, seed=61, scale=10.0)
    batch = O.synthetic_batch(cfg, B=4, T=32, seed=62)
    _, rec = check_grads(cfg, params, batch)
    plan = rec.decoder_plan()
    print("PLAN", case, plan)
    assert plan["ran"] == (case == "c512"), plan


def test_training_steps_match_oracle_c512():
    """Two optimizer steps (momentum + AdaDelta + max-norm) with dim_dec 512 and a Maxout(4) readout."""
    _torch()
    cfg = _config("c512")
    params = O.init_params(cfg, seed=71, scale=10.0)
    tc = G.make_train_config(gradient_threshold=2.0, rules=("momentum", "adadelta"), scale=0.05, momentum=0.5,
                             decay_rate=0.95, epsilon=1e-6, max_norm=1.0)
    train_like_the_oracle(cfg, params, tc, B=4, T=32)


# ---- refusals ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("net,message", [
    (dict(dim_dec=250), "multiples of 8"),                         # the reference's wsj_paper* / wsj_prior_conv width
    (dict(post_merge_dims=[250]), "multiples of 8"),
    (dict(dim_output_embedding=250), "dim_feedback must be a multiple of 4"),
    (dict(post_merge_dims=[256], maxout_pieces=3), "bad maxout_pieces"),
], ids=["dim_dec_250", "post_merge_250", "feedback_250", "maxout3_over_256"])
def test_widths_beyond_the_kernels_are_refused(net, message):
    _torch()
    cfg = O.make_config(**dict(PYRAMID, **net))
    with pytest.raises((ValueError, RuntimeError), match=message):
        make_recognizer(cfg, O.init_params(cfg, seed=1, scale=10.0))
