"""The persistent (island-mode) decoder at the exact shapes bench.py times, against the float64
oracle: committed golden fixtures for the BASELINE metric config (B=64 x T=1000, L=125) and
config 2 (B=32 x T=800, L=100) -- tests/golden/make_metric_golden.py -- and live oracle runs at
island-mode batch sizes for every window prior.  Tolerance 1e-4 relative (BASELINE north_star)."""
import os

import numpy as np
import pytest

import bench
from helpers import O, PYRAMID, make_recognizer, package, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _projections(E, C, Tp, seed=99):          # same draws as tests/golden/make_metric_golden.py
    rng = np.random.RandomState(seed)
    return dict(pE=rng.normal(size=E), pC=rng.normal(size=C), pT=rng.normal(size=Tp))


@pytest.mark.parametrize("name,B,T,L", [("metric", 64, 1000, 125), ("config2", 32, 800, 100)])
def test_benchmarked_shapes_match_float64_oracle(name, B, T, L, monkeypatch):
    torch = _torch()
    monkeypatch.setenv("LVSR_DEC_CHECK", "1")      # post-condition: launch status 0, no sentinel word left
    gold = np.load(os.path.join(GOLDEN, "%s_golden.npz" % name))
    cfg = O.make_config(**bench.NET)
    rec = make_recognizer(cfg)
    rec.set_parameter_values(bench.init_values(rec.parameter_shapes()))
    x, m, labels, lm = bench.synthetic_batch(B, T, 40, L, 32, seed=1234)
    att, attm = rec.encode(x, m)
    proj = _projections(att.shape[2], cfg["dim_dec"], att.shape[0])
    errs = {"attended": rel_err(att.double().cpu().numpy().dot(proj["pE"]), gold["attended_p"])}
    r = rec.cost_matrix(labels, lm, att, attm, return_all=True)
    status, fallbacks = rec.launch_status()
    assert status == 0 and fallbacks == 0
    plan = rec.decoder_plan()
    assert plan["ran"] and plan["nisl"] == B // 16, plan
    g = {k: v.double().cpu().numpy() for k, v in r.items()}
    errs["costs"] = rel_err(g["costs"], gold["costs"])
    errs["states"] = rel_err(g["states"].dot(proj["pC"]), gold["states_p"])
    errs["weighted_averages"] = rel_err(g["weighted_averages"].dot(proj["pE"]), gold["wavg_p"])
    errs["weights"] = rel_err(g["weights"].dot(proj["pT"]), gold["weights_p"])
    errs["energies"] = rel_err(g["energies"].dot(proj["pT"]), gold["energies_p"])
    print(name, errs)
    for k, e in errs.items():
        assert e < TOL, (k, e)
    # identical argmax of the alignment wherever the oracle's top two weights are not a near tie
    w = g["weights"]
    top2 = np.sort(w, axis=-1)[..., -2:]
    clear = (top2[..., 1] - top2[..., 0]) > 1e-4
    assert np.array_equal(w.argmax(-1)[clear], gold["weights_argmax"][clear])
    # the host-buffer entry point (what bench.py's e2e times) returns the same costs
    host = rec.cost(x, m, labels, lm)
    assert rel_err(host, gold["costs"]) < TOL
    assert rec.launch_status() == (0, 0)


PRIORS = [
    dict(type="expanding", initial_begin=0, initial_end=10000, min_speed=0, max_speed=0),
    dict(type="expanding", initial_begin=0, initial_end=8, min_speed=0.6, max_speed=1.9),
    dict(type="window_around_median", before=7, after=9),
    dict(type="window_around_mean", before=8, after=8),
]


@pytest.mark.parametrize("prior", PRIORS, ids=lambda p: p["type"] + str(p.get("initial_end", p.get("before"))))
@pytest.mark.parametrize("B", [16, 37, 64])
def test_island_mode_matches_oracle(prior, B, monkeypatch):
    """B >= 16 runs the persistent decoder in island mode (dec_scan.cu): 1, 3 and 4 islands, ragged island sizes
    (37 = 13+12+12), every window prior.  T' = 32 lets the planner choose 2-CTA clusters; at cs 1 the 12-row islands
    of B = 37 have too few CTAs for the dense tiles and the planner would take the global layout instead."""
    _torch()
    monkeypatch.setenv("LVSR_DEC_CHECK", "1")
    cfg = O.make_config(prior=prior, **PYRAMID)
    params = O.init_params(cfg, seed=8, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=B, T=128, seed=31 + B)
    att, attm = O.encoder(cfg, params, x, m)
    want = O.cost_matrix(cfg, params, att, attm, labels, lm, return_all=True)
    rec = make_recognizer(cfg, params)
    got = rec.cost_matrix(labels, lm, att.astype(np.float32), attm.astype(np.float32), return_all=True)
    assert rec.launch_status() == (0, 0)
    plan = rec.decoder_plan()
    assert plan["ran"] and plan["cs"] == 2 and plan["nisl"] == -(-B // 16) and plan["grid"] == 2 * B, plan
    errs = {k: rel_err(got[k].cpu().numpy(), want[k]) for k in
            ("costs", "weights", "energies", "states", "weighted_averages")}
    print(prior["type"], B, errs)
    for k, e in errs.items():
        assert e < TOL, (k, e)


def test_smoke_passes_with_decoder_postcondition(monkeypatch):
    """__graft_entry__.smoke() with the debug post-condition of the persistent decoder on."""
    _torch()
    monkeypatch.setenv("LVSR_DEC_CHECK", "1")
    import __graft_entry__ as g
    g.smoke()


def test_long_utterance_persistent_decoder_matches_oracle(monkeypatch):
    """16 rows x T' = 1600 (the shape class of BASELINE config 5): 4-CTA clusters with 400-position chunks; the dense
    tiles' scratch shares the attention scratch so that the persistent kernel fits in shared memory."""
    _torch()
    monkeypatch.setenv("LVSR_DEC_CHECK", "1")
    net = dict(num_features=40, dims_bidir=[128], subsample=[1], dim_dec=128, dim_matcher=256, conv_n=50,
               conv_num_filters=10, num_phonemes=32, post_merge_dims=[128], maxout_pieces=2)
    cfg = O.make_config(prior=dict(type="window_around_median", before=60, after=60), **net)
    params = O.init_params(cfg, seed=8, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=16, T=1600, seed=3, label_div=100)
    att, attm = O.encoder(cfg, params, x, m)
    want = O.cost_matrix(cfg, params, att, attm, labels, lm, return_all=True)
    rec = make_recognizer(cfg, params)
    import ctypes as C
    pkg = package()
    lib = pkg._lib.load()
    lib.lvsr_profile_enable(1)
    got = rec.cost_matrix(labels, lm, att.astype(np.float32), attm.astype(np.float32), return_all=True)
    tot, cnt = C.c_double(), C.c_int64()
    lib.lvsr_profile_read(b"attention", C.byref(tot), C.byref(cnt))
    lib.lvsr_profile_enable(0)
    assert cnt.value == 0, "the step-wise fallback ran instead of the persistent decoder"
    assert rec.launch_status() == (0, 0)
    plan = rec.decoder_plan()
    assert plan["ran"] and plan["cs"] == 4 and plan["nisl"] == 1 and plan["red_alias"] == 1, plan
    for k in ("costs", "weights", "energies", "states", "weighted_averages"):
        assert rel_err(got[k].cpu().numpy(), want[k]) < TOL, k
