"""CUDA path vs the float64 oracle on the same seeded inputs (run on an H100).

Bar (BASELINE.json north_star): forward activations within 1e-4 relative of the
reference math, identical argmax / beam token sequences.  Everything goes through the
C ABI (ctypes -> liblvsr_b200.so).
"""
import numpy as np
import pytest

from helpers import O, PYRAMID, SMALL, WSJ, make_recognizer, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


@pytest.mark.parametrize("name,net,B,T,use_mask", [
    ("small_mask", SMALL, 5, 37, True),
    ("small_nomask", SMALL, 8, 40, False),
    ("pyramid_mask", PYRAMID, 11, 61, True),
    ("single_utt", PYRAMID, 1, 50, False),
])
def test_encoder_matches_oracle(name, net, B, T, use_mask):
    _torch()
    cfg = O.make_config(**net)
    params = O.init_params(cfg, seed=3, scale=10.0)
    x, m, _, _ = O.synthetic_batch(cfg, B, T, seed=11)
    want, want_mask = O.encoder(cfg, params, x, m if use_mask else None)
    rec = make_recognizer(cfg, params)
    got, got_mask = rec.encode(x, m if use_mask else None)
    assert tuple(got.shape) == want.shape
    err = rel_err(got.cpu().numpy(), want)
    print(name, "encoder rel err", err)
    assert err < TOL
    assert np.array_equal(got_mask.cpu().numpy(), want_mask.astype(np.float32))


PRIORS = [
    dict(type="expanding", initial_begin=0, initial_end=10000, min_speed=0, max_speed=0),
    dict(type="expanding", initial_begin=0, initial_end=6, min_speed=0.7, max_speed=2.2),
    dict(type="window_around_median", before=5, after=7),
    dict(type="window_around_mean", before=6, after=6),
]


@pytest.mark.parametrize("prior", PRIORS, ids=lambda p: p["type"] + str(p.get("initial_end", p.get("before"))))
@pytest.mark.parametrize("normalizer", ["softmax", "logistic", "relu"])
def test_cost_matrix_matches_oracle(prior, normalizer):
    _torch()
    cfg = O.make_config(prior=prior, energy_normalizer=normalizer, **PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    if normalizer != "softmax":
        # keeps relu energies positive: an all-zero relu column is 0/0 = NaN in the reference too
        params["/recognizer/generator/att_trans/conv_att/energy_comp/linear.b"][:] = 3.0
    x, m, labels, lm = O.synthetic_batch(cfg, B=6, T=88, seed=21)
    att, attm = O.encoder(cfg, params, x, m)
    want = O.cost_matrix(cfg, params, att, attm, labels, lm, return_all=True)
    rec = make_recognizer(cfg, params)
    got = rec.cost_matrix(labels, lm, att.astype(np.float32), attm.astype(np.float32), return_all=True)
    errs = {k: rel_err(got[k].cpu().numpy(), want[k]) for k in
            ("costs", "weights", "energies", "states", "weighted_averages")}
    print(prior["type"], normalizer, errs)
    for k, e in errs.items():
        assert e < TOL, (k, e)


def test_recognizer_cost_host_path_and_analyze():
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=9, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=7, T=72, seed=4)
    want = O.recognizer_cost(cfg, params, x, m, labels, lm)
    rec = make_recognizer(cfg, params)
    got = rec.cost(x, m, labels, lm)                      # host buffers through lvsr_recognizer_cost_host
    assert rel_err(got, want) < TOL
    # masked costs are exactly zero
    assert np.all(got[lm == 0] == 0)
    # analyze: batch of one, no masks
    c, w, e = rec.analyze({"recordings": x[:, 0, :]}, labels[:, 0])
    wc, ww, we = O.analyze(cfg, params, x[:, 0, :], labels[:, 0])
    assert rel_err(c, wc) < TOL and rel_err(w, ww) < TOL and rel_err(e, we) < TOL
    assert np.allclose(w.sum(axis=1), 1.0, atol=1e-5)


def _np_states(st):
    return {k: v.cpu().numpy() for k, v in st.items()}


def test_generate_step_functions_match_oracle():
    torch = _torch()
    cfg = O.make_config(prior=dict(type="window_around_median", before=6, after=8), **PYRAMID)
    params = O.init_params(cfg, seed=13, scale=10.0)
    x, _, _, _ = O.synthetic_batch(cfg, B=3, T=64, seed=2)
    att, attm = O.context_computer(cfg, params, x)
    rec = make_recognizer(cfg, params)
    g_att, g_attm = rec.encode(x, None)
    assert rel_err(g_att.cpu().numpy(), att) < TOL
    ctx = dict(attended=g_att, attended_mask=g_attm)      # preprocessed omitted: recomputed like the reference
    st_o = O.initial_states(cfg, params, 3, att)
    st_g = rec._initial_states(att.shape[0], 3)
    for k in st_o:
        assert np.allclose(st_g[k].cpu().numpy(), st_o[k], atol=1e-6), k
    for step in range(6):
        lp_o = O.logprobs_computer(cfg, params, att, attm, st_o)
        lp_g = rec._logprobs(ctx, st_g).cpu().numpy()
        assert rel_err(lp_g, lp_o) < TOL
        y = lp_o.argmin(axis=1)
        assert np.array_equal(lp_g.argmin(axis=1), y)
        st_o = O.next_state_computer(cfg, params, att, attm, st_o, y)
        st_g = rec._next_states(ctx, st_g, y)
        for k in ("states", "weighted_averages", "weights", "energies"):
            assert rel_err(st_g[k].cpu().numpy(), st_o[k]) < TOL, (step, k)
        assert np.array_equal(st_g["step"].cpu().numpy(), st_o["step"])


@pytest.mark.parametrize("beam_size,stop_on,char_discount", [(1, "patience", 0), (4, "patience", 0),
                                                            (10, "optimistic_future_cost", 0.1)])
def test_beam_search_tokens_identical(beam_size, stop_on, char_discount):
    _torch()
    cfg = O.make_config(max_decoded_length_scale=2.0, **PYRAMID)
    params = O.init_params(cfg, seed=17, scale=10.0)
    # "trained-like": peaky output distribution, eos competitive so hypotheses finish
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.W"] *= 40
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.b"][cfg["eos_label"]] = 24.0
    rec = make_recognizer(cfg, params)
    rec.init_beam_search(beam_size)
    rng = np.random.RandomState(0)
    for utt in range(3):
        x = rng.normal(size=(40 + 8 * utt, cfg["num_features"]))
        pkg_err = type(rec._beam_search).__module__
        try:
            want_out, want_costs = O.beam_search(cfg, params, x, beam_size, stop_on=stop_on,
                                                 char_discount=char_discount)
        except O.CandidateNotFoundError:
            # greedy search that never emits eos: the CUDA path must fail the same way
            import sys
            with pytest.raises(sys.modules[pkg_err].CandidateNotFoundError):
                rec.beam_search({"recordings": x}, stop_on=stop_on, char_discount=char_discount)
            continue
        got_out, got_costs = rec.beam_search({"recordings": x}, stop_on=stop_on, char_discount=char_discount)
        assert got_out == want_out
        assert np.allclose(got_costs, want_costs, rtol=1e-4, atol=1e-4)


def test_wsj_shape_slice_matches_oracle():
    """The BASELINE architecture (4x BiGRU(256) pyramid, M=512, K=10, n=100) on a batch the
    float64 oracle finishes in seconds."""
    _torch()
    cfg = O.make_config(**WSJ)
    params = O.init_params(cfg, seed=1, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=4, T=120, seed=1234)
    want = O.recognizer_cost(cfg, params, x, m, labels, lm, return_all=True)
    rec = make_recognizer(cfg, params)
    att, attm = rec.encode(x, m)
    o_att, _ = O.encoder(cfg, params, x, m)
    e_enc = rel_err(att.cpu().numpy(), o_att)
    got = rec.cost_matrix(labels, lm, att, attm, return_all=True)
    errs = {k: rel_err(got[k].cpu().numpy(), want[k]) for k in ("costs", "weights", "states", "weighted_averages")}
    print("wsj slice: encoder", e_enc, errs)
    assert e_enc < TOL
    for k, e in errs.items():
        assert e < TOL, (k, e)


def test_full_size_properties():
    """BASELINE metric shape (B=64, T=1000): size-independent properties instead of the oracle."""
    torch = _torch()
    cfg = O.make_config(**WSJ)
    params = O.init_params(cfg, seed=1, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=64, T=1000, seed=1234, dtype=np.float32)
    rec = make_recognizer(cfg, params)
    att, attm = rec.encode(x, m)
    assert tuple(att.shape) == (250, 64, 512) and bool(torch.isfinite(att).all())
    r = rec.cost_matrix(labels, lm, att, attm, return_all=True)
    w = r["weights"]
    assert bool(torch.isfinite(r["costs"]).all())
    assert torch.allclose(w.sum(dim=2), torch.ones_like(w.sum(dim=2)), atol=1e-4)       # weights sum to 1
    assert float((w * (1 - attm.T[None])).abs().max()) == 0.0                            # zero where the mask is 0
    assert float(r["costs"][torch.as_tensor(lm) == 0].abs().max()) == 0.0
    # batch independence: utterance 5 alone gives the same costs as inside the batch
    sub = rec.cost(x[:, 5:6], m[:, 5:6], labels[:, 5:6], lm[:, 5:6])
    assert rel_err(sub[:, 0], r["costs"][:, 5].cpu().numpy()) < 1e-4


# ---- BASELINE.json configs as parity cases -------------------------------------------------

def _peaky(cfg, seed, gain=40.0, eos_bias=24.0):
    params = O.init_params(cfg, seed=seed, scale=10.0)
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.W"] *= gain
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.b"][cfg["eos_label"]] = eos_bias
    return params


def test_config1_greedy_decode_identical_tokens():
    """configs[0]: 8 utterances x 200 frames x 40 fbank, 1-layer BiGRU(128), greedy decode."""
    _torch()
    cfg = O.make_config(num_features=40, dims_bidir=[128], subsample=[1], dim_dec=128, conv_n=100,
                        conv_num_filters=10, num_phonemes=32, post_merge_dims=[128], maxout_pieces=2,
                        max_decoded_length_scale=8.0)
    params = _peaky(cfg, 3, eos_bias=4.0)
    x, m, _, _ = O.synthetic_batch(cfg, B=8, T=200, seed=1234)
    rec = make_recognizer(cfg, params)
    # batched greedy generate (argmax emission) through the state functions, all 8 utterances at once
    att_o, attm_o = O.encoder(cfg, params, x, m)
    ys_o, costs_o, _ = O.generate_greedy(cfg, params, att_o, attm_o, 25)
    att, attm = rec.encode(x, m)
    ctx = dict(attended=att, attended_mask=attm, preprocessed=rec.preprocess(att))
    st = rec._initial_states(att.shape[0], 8)
    ys = []
    for _ in range(25):
        lp = rec._logprobs(ctx, st).cpu().numpy()
        y = lp.argmin(axis=1)
        ys.append(y)
        st = rec._next_states(ctx, st, y)
    assert np.array_equal(np.stack(ys), ys_o)
    # and beam_size = 1 search of single utterances
    rec.init_beam_search(1)
    for b in range(2):
        n = int(m[:, b].sum())
        try:
            want = O.beam_search(cfg, params, x[:n, b], 1)
        except O.CandidateNotFoundError:
            import sys
            err = sys.modules[type(rec._beam_search).__module__].CandidateNotFoundError
            with pytest.raises(err):
                rec.beam_search({"recordings": x[:n, b]})
            continue
        got = rec.beam_search({"recordings": x[:n, b]})
        assert got[0] == want[0]


def test_config3_wsj_beam10_identical_tokens():
    """configs[2]: WSJ architecture, beam_size = 10, char-level output (short utterance so the
    float64 oracle search finishes in seconds)."""
    _torch()
    cfg = O.make_config(max_decoded_length_scale=6.0, **WSJ)
    params = _peaky(cfg, 5)
    rng = np.random.RandomState(4)
    x = rng.normal(size=(160, cfg["num_features"]))
    want_out, want_costs = O.beam_search(cfg, params, x, 10, stop_on="optimistic_future_cost", char_discount=0.1)
    rec = make_recognizer(cfg, params)
    rec.init_beam_search(10)
    got_out, got_costs = rec.beam_search({"recordings": x}, stop_on="optimistic_future_cost", char_discount=0.1)
    assert got_out == want_out
    # the x40 readout gain makes the logits ~25 in magnitude: 1e-4 relative on them is ~2.5e-3 absolute per token
    assert np.allclose(got_costs, want_costs, rtol=1e-3, atol=5e-3)


def test_persistent_decoder_equals_stepwise_kernels(monkeypatch):
    _torch()
    cfg = O.make_config(prior=dict(type="window_around_mean", before=9, after=9), **PYRAMID)
    params = O.init_params(cfg, seed=8, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=9, T=80, seed=9)
    rec = make_recognizer(cfg, params)
    att, attm = rec.encode(x, m)
    a = rec.cost_matrix(labels, lm, att, attm, return_all=True)
    assert rec.decoder_plan()["ran"]
    monkeypatch.setenv("LVSR_NO_DEC_SCAN", "1")
    b = rec.cost_matrix(labels, lm, att, attm, return_all=True)
    assert not rec.decoder_plan()["ran"]
    for k in ("costs", "weights", "energies", "states", "weighted_averages"):
        assert rel_err(a[k].cpu().numpy(), b[k].cpu().numpy()) < 2e-5, k


def test_tensor_core_gemm_equals_fp32_tiles(monkeypatch):
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=10, scale=10.0)
    x, m, _, _ = O.synthetic_batch(cfg, B=10, T=90, seed=11)
    rec_tc = make_recognizer(cfg, params)
    a, _ = rec_tc.encode(x, m)
    pa = rec_tc.preprocess(a)
    monkeypatch.setenv("LVSR_NO_TC_GEMM", "1")
    rec_simt = make_recognizer(cfg, params)        # the switch is read at finalize
    b, _ = rec_simt.encode(x, m)
    pb = rec_simt.preprocess(b)
    assert rel_err(a.cpu().numpy(), b.cpu().numpy()) < 1e-5
    assert rel_err(pa.cpu().numpy(), pb.cpu().numpy()) < 1e-5
