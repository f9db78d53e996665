"""The projection of encoder layer l + 1 streamed beside the BiGRU scan of layer l (csrc/gemm_tc.cu:
gemm_f16_stream_kernel, csrc/api.cu: run_encoder).  Every tile is computed as the projection after the scan computes
it, so the encoder output must be bit-identical with LVSR_ENC_OVERLAP=0, whichever launch did which tile; each case
asserts through encoder_plan() where the overlap ran and that the two launches together did every tile once."""
import numpy as np
import pytest

import unidirectional_oracle as U
from helpers import O, WSJ, check_grads, f32, make_recognizer
from helpers import check_overlap_claims as _check_claims

pytestmark = pytest.mark.gpu


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _encode(rec, x, m):
    att, attm = rec.encode(x, m)
    return att.cpu().numpy(), attm.cpu().numpy(), rec.encoder_plan()


def _case(net, B, T, seed, monkeypatch, one_frame=False, spin_limit=None, warm=False, reps=1, bidir=True):
    """encode with the overlap on and off: bit-identical outputs; returns the plan of the last run with the overlap on.

    The workspace persists across calls at the same offsets in both modes, so before every overlap-on run the test
    encodes a decoy batch of the same shape (overlap off): the scan outputs, split planes, exponents and pre-activations
    the streamed projection reads and writes then hold another batch's values, and a tile read before its rows are final
    or never written shows in the output; and each tile claimed beside a scan must have been claimed at a progress that
    makes its rows final (_check_claims).  warm: the first call of all has the overlap on (its launch beside the scan
    also loads the streamed kernel's module) and is compared too; reps: decoy + overlap-on runs; bidir False: the
    forward-only encoder (tests/unidirectional_oracle.py's parameters), whose projections have 3 D columns."""
    _torch()
    M = O if bidir else U
    ndir = 2 if bidir else 1
    cfg = M.make_config(**dict(WSJ, **net))
    rec = make_recognizer(cfg, M.init_params(cfg, seed=seed, scale=10.0), bidir=bidir)
    x, m, _, _ = O.synthetic_batch(cfg, B=B, T=T, seed=seed + 1)
    decoy = O.synthetic_batch(cfg, B=B, T=T, seed=seed + 2)[0]
    if one_frame:
        m[1:, 0] = 0.0                                    # row 0 is a one-frame utterance
    runs = []
    if warm:
        runs.append(_encode(rec, x, m))
        _check_claims(rec, runs[-1][2], B, cfg["subsample"], ndir)
    monkeypatch.setenv("LVSR_ENC_OVERLAP", "0")
    want, wantm, off = _encode(rec, x, m)
    assert not any(p["overlap"] for p in off), off
    if spin_limit is not None:
        monkeypatch.setenv("LVSR_ENC_OVERLAP_SPIN_LIMIT", str(spin_limit))
    for _ in range(reps):
        monkeypatch.setenv("LVSR_ENC_OVERLAP", "0")
        rec.encode(decoy, m)
        monkeypatch.delenv("LVSR_ENC_OVERLAP")
        runs.append(_encode(rec, x, m))
        _check_claims(rec, runs[-1][2], B, cfg["subsample"], ndir)
    dims = cfg["dims_bidir"]
    for got, gotm, plan in runs:
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.abs(got - want).max()
        assert np.array_equal(gotm, wantm)
        for l, p in enumerate(plan):
            assert (p["proj"], p["operands"]) == (off[l]["proj"], off[l]["operands"]), (l, p, off[l])
            if p["overlap"]:
                # 128 x 128 output tiles: ceil(T_l B / 128) row tiles x 3 ndir D_l / 128 column tiles
                tiles = -(-p["T"] * B // 128) * (3 * ndir * dims[l] // 128)
                assert p["tiles_beside"] + p["tiles_after"] == tiles, (l, p, tiles)
            else:
                assert p["tiles_beside"] == p["tiles_after"] == 0, (l, p)
        print("B=%d T=%d" % (B, T), [(p["overlap"], p["tiles_beside"], p["tiles_after"]) for p in plan])
    return runs[-1][2]


def test_metric_shape(monkeypatch):
    """B = 64, T = 1000 on the benchmarked encoder: one wave of 16 eight-row clusters (64 SMs), the projections of
    layers 1-3 run beside the scans and do part of their tiles there"""
    plan = _case({}, 64, 1000, 1, monkeypatch, warm=True, reps=3)
    assert [p["overlap"] for p in plan] == [False, True, True, True], plan
    assert all(p["tiles_beside"] > 0 for p in plan[1:]), plan


def test_tile_ending_on_a_publication_boundary(monkeypatch):
    """The scan publishes its progress every 16 steps, so a readiness rule off by one frame only claims a tile too early
    when the tile's last frame lands on a publication.  B = 17, T = 160: m-tile 14 holds frames 105..112, needs forward
    progress 113, and becomes ready, with the tiles claimed before it, when the progress reaches 128; a rule one frame
    short claims it at 112.  At 17 rows the projection keeps up with the scan, so the tile is claimed at the first
    progress the rule accepts."""
    plan = _case(dict(dims_bidir=[256, 256], subsample=[1, 1]), 17, 160, 70, monkeypatch, warm=True, reps=3)
    assert [p["overlap"] for p in plan] == [False, True] and plan[1]["tiles_beside"] > 0, plan


@pytest.mark.parametrize("B", [1, 3, 33])
def test_tiles_straddling_frames(B, monkeypatch):
    """128-row tiles hold parts of several frames when B does not divide 128; B = 33 also holds a one-frame utterance"""
    plan = _case({}, B, 61, 10 + B, monkeypatch, one_frame=B > 1)
    assert [p["overlap"] for p in plan] == [False, True, True, True], plan


@pytest.mark.parametrize("subsample,T", [([1, 3], 62), ([2, 2, 2], 61)], ids=["1-3", "2-2-2"])
def test_subsampling(subsample, T, monkeypatch):
    net = dict(dims_bidir=[256] * len(subsample), subsample=subsample)
    plan = _case(net, 5, T, 20 + T, monkeypatch, one_frame=True)
    assert [p["overlap"] for p in plan] == [False] + [True] * (len(subsample) - 1), plan


def test_one_frame_utterance_batch(monkeypatch):
    """T = 1: the scan has one step, the projection behind it one frame"""
    plan = _case(dict(dims_bidir=[256, 256], subsample=[1, 1]), 4, 1, 30, monkeypatch)
    assert [p["overlap"] for p in plan] == [False, True], plan


def test_mixed_widths(monkeypatch):
    """[256, 128, 256]: the scan of layer 0 (tensor cores) takes the 128-wide layer 1's projection beside it; the
    128-wide scan (FFMA kernel) publishes no progress, so layer 2's projection runs after it"""
    plan = _case(dict(dims_bidir=[256, 128, 256], subsample=[1, 1, 1]), 6, 40, 31, monkeypatch)
    assert [p["overlap"] for p in plan] == [False, True, False], plan
    assert [p["bigru"] for p in plan] == ["mma", "ffma", "mma"], plan


def test_two_scan_waves_decline_the_overlap(monkeypatch):
    """a batch that needs two waves of clusters: no SM is idle beside the scan, the projection runs after it"""
    cfg = dict(dims_bidir=[256, 256], subsample=[1, 1])
    plan = _case(cfg, 1, 8, 40, monkeypatch)
    resident = plan[0]["resident"]
    B = 8 * (resident // 2 + 1)                            # 2 * ceil(B / 8) > resident, for 4- and 8-row clusters
    plan = _case(cfg, B, 8, 41, monkeypatch)
    assert plan[0]["waves"] >= 2 and [p["overlap"] for p in plan] == [False, False], plan


def test_spin_limit_zero_leaves_every_tile_to_the_launch_after_the_scan(monkeypatch):
    """LVSR_ENC_OVERLAP_SPIN_LIMIT=0: beside the scan, the first tile whose rows are not final ends the claiming; at
    the start of a 400-step scan no row is final, so the launch after the scan does every tile (warm: the streamed
    kernel's module is loaded before, so the launch beside the scan starts while the scan does)"""
    plan = _case({}, 16, 400, 50, monkeypatch, spin_limit=0, warm=True)
    assert [p["overlap"] for p in plan] == [False, True, True, True], plan
    assert all(p["tiles_beside"] == 0 for p in plan[1:]), plan


def test_training_forward_overlaps_and_matches_the_gradient_oracle():
    """the training forward (with the scans' tape) takes the same path; cost and gradients against the float64 oracle"""
    _torch()
    cfg = O.make_config(**dict(WSJ, dims_bidir=[256, 256], subsample=[1, 2], dim_matcher=256))
    params = O.init_params(cfg, seed=60, scale=10.0)
    params = {k: f32(v) for k, v in params.items()}
    x, m, labels, lm = O.synthetic_batch(cfg, B=5, T=40, seed=61)
    _, rec = check_grads(cfg, params, (f32(x), m, labels, lm))
    plan = rec.encoder_plan()
    assert [(p["overlap"], p["tape"]) for p in plan] == [(False, True), (True, True)], plan
    _check_claims(rec, plan, 5, cfg["subsample"])
    assert plan[1]["tiles_beside"] + plan[1]["tiles_after"] == -(-40 * 5 // 128) * 12, plan
