"""The projection of encoder layer l + 1 streamed beside the forward-only scan of layer l (net.bidir: False): every case
of test_gpu_encoder_overlap.py restated with one direction, through its _case (a decoy batch before every overlap-on
run, the output bit-identical with LVSR_ENC_OVERLAP=0, every claimed tile's rows final at the forward progress it was
claimed at and no backward progress recorded, ceil(T_l B / 128) * 3 D_l / 128 tiles done once between the two launches);
where the overlap declines with one direction; and the order the launch beside the scan claims its m-tiles in.

With one direction an input frame f of layer l + 1 is final once the scan has stored step f k, so rows become final
from frame 0 upward and gemm_f16_stream claims m-tile 0 first, then upward (mid = 0); with two directions it claims the
middle m-tile first, where the two scans meet, then outward.  test_claim_order pins both.

Measured on an H100 80GB HBM3 (700 W power limit): at B = 64, T = 1000 the launch beside the forward-only scans did
2996 of 3000, 2996 of 3000 and 1500 of 1500 tiles of layers 1-3 (the bidirectional encoder: 4416 of 6000, 4412 of 6000,
2982 of 3000); the card holds 30 four-CTA clusters, so B = 240 leaves 12 SMs free and the overlap declines; the training
forward's worst gradient error was 8.9e-6 of a parameter's largest entry (bar 1e-4).  The file runs in about 15 s."""
import numpy as np
import pytest

import unidirectional_oracle as U
from helpers import O, WSJ, check_overlap_claim_order, check_overlap_claims, check_unidirectional_grads, f32
from helpers import make_recognizer
from test_gpu_encoder_overlap import _case as _bi_case

pytestmark = pytest.mark.gpu

ENC_OVERLAP_MIN_SMS = 16      # api.cu: SMs the scan must leave free for the launch beside it


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _case(net, B, T, seed, monkeypatch, **kw):
    return _bi_case(net, B, T, seed, monkeypatch, bidir=False, **kw)


def test_metric_shape(monkeypatch):
    """B = 64, T = 1000 on bench.NET's forward-only encoder: one wave of 16 four-row clusters (64 SMs), the projections
    of layers 1-3 run beside the scans and do part of their tiles there"""
    plan = _case({}, 64, 1000, 1, monkeypatch, warm=True, reps=3)
    assert [p["overlap"] for p in plan] == [False, True, True, True], plan
    assert (plan[0]["rb"], plan[0]["clusters"], plan[0]["waves"]) == (4, 16, 1), plan[0]
    assert all(p["tiles_beside"] > 0 for p in plan[1:]), plan


def test_tile_ending_on_a_publication_boundary(monkeypatch):
    """The scan publishes its progress every 16 steps.  B = 17, T = 160: m-tile 14 holds rows 1792..1919, frames
    105 (1792 // 17) to 112 (1919 // 17), so with one direction it needs forward progress 113 and is claimable at the
    publication of 128; a rule one frame short would claim it at 112, itself a publication.  Claims ascend from
    m-tile 0 here, and at 17 rows the projection keeps up with the scan, so every tile is claimed at the first progress
    the rule accepts."""
    plan = _case(dict(dims_bidir=[256, 256], subsample=[1, 1]), 17, 160, 70, monkeypatch, warm=True, reps=3)
    assert [p["overlap"] for p in plan] == [False, True] and plan[1]["tiles_beside"] > 0, plan
    assert (14 * 128) // 17 == 105 and (15 * 128 - 1) // 17 == 112


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
    """[256, 128, 256]: the tensor-core scan of layer 0 takes the 128-wide layer 1's projection (3 D = 384 columns,
    fp16) beside it; the 128-wide scan (FFMA kernel) publishes no progress, so layer 2's projection runs after it"""
    plan = _case(dict(dims_bidir=[256, 128, 256], subsample=[1, 1, 1]), 6, 40, 31, monkeypatch)
    assert [p["overlap"] for p in plan] == [False, True, False], plan
    assert [p["bigru"] for p in plan] == ["mma", "ffma", "mma"], plan


def test_spin_limit_zero_leaves_every_tile_to_the_launch_after_the_scan(monkeypatch):
    """LVSR_ENC_OVERLAP_SPIN_LIMIT=0: beside the scan, the first tile whose rows are not final ends the claiming; at
    the start of a 400-step scan no row is final, so the launch after the scan does every tile"""
    plan = _case({}, 16, 400, 50, monkeypatch, spin_limit=0, warm=True)
    assert [p["overlap"] for p in plan] == [False, True, True, True], plan
    assert all(p["tiles_beside"] == 0 for p in plan[1:]), plan


def test_training_forward_overlaps_and_matches_the_gradient_oracle():
    """the training forward (with the scans' tape) takes the same path; cost and gradients against the float64
    oracle of tests/unidirectional_oracle.py"""
    _torch()
    cfg = U.make_config(**dict(WSJ, dims_bidir=[256, 256], subsample=[1, 2], dim_matcher=256))
    params = {k: f32(v) for k, v in U.init_params(cfg, seed=60, scale=10.0).items()}
    x, m, labels, lm = O.synthetic_batch(cfg, B=5, T=40, seed=61)
    rec = check_unidirectional_grads(cfg, params, (f32(x), m, labels, lm))
    plan = rec.encoder_plan()
    assert [(p["overlap"], p["tape"]) for p in plan] == [(False, True), (True, True)], plan
    check_overlap_claims(rec, plan, 5, cfg["subsample"], ndir=1)
    assert plan[1]["tiles_beside"] + plan[1]["tiles_after"] == -(-40 * 5 // 128) * 6, plan


# ---- where the overlap declines -------------------------------------------------------------------------------------

def test_two_scan_waves_decline_the_overlap(monkeypatch):
    """One direction needs ceil(B / rb) clusters.  Forced 4-row clusters: B = 4 (resident + 1) is the smallest batch
    that needs two waves; as planned (8-row clusters, which take over once 4-row ones need more waves), B =
    8 (resident + 1).  No SM is idle beside the scan, so the projection runs after it."""
    cfg = dict(dims_bidir=[256, 256], subsample=[1, 1])
    for rb in (4, 8):
        monkeypatch.setenv("LVSR_BIGRU_RB", str(rb))
        plan = _case(cfg, 1, 8, 40, monkeypatch)
        resident = plan[0]["resident"]
        B = rb * (resident + 1)
        if rb == 8:
            monkeypatch.delenv("LVSR_BIGRU_RB")
        plan = _case(cfg, B, 8, 41 + rb, monkeypatch)
        p = plan[0]
        assert (p["rb"], p["clusters"], p["resident"]) == (rb, resident + 1, resident), p
        assert p["waves"] == 2 and [q["overlap"] for q in plan] == [False, False], plan


def test_one_wave_without_enough_free_sms_declines_the_overlap(monkeypatch):
    """One wave of c four-CTA clusters leaves SMs - 4 c free; below ENC_OVERLAP_MIN_SMS = 16 the projection runs after
    the scan.  B = 8 resident (8-row clusters, as planned: 4-row ones would need two waves) is the fullest one-wave
    batch; an H100 that holds too few clusters for it to leave fewer than 16 SMs free cannot reach this case."""
    torch = _torch()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cfg = dict(dims_bidir=[256, 256], subsample=[1, 1])
    resident = _case(cfg, 1, 8, 40, monkeypatch)[0]["resident"]
    if sms - 4 * resident >= ENC_OVERLAP_MIN_SMS:
        pytest.skip("%d SMs hold %d four-CTA clusters: one wave leaves at least %d SMs free"
                    % (sms, resident, sms - 4 * resident))
    B = 8 * resident
    plan = _case(cfg, B, 8, 42, monkeypatch)
    p = plan[0]
    print("%d SMs, %d clusters resident, B = %d: %d SMs free" % (sms, resident, B, sms - 4 * p["clusters"]))
    assert (p["rb"], p["clusters"], p["waves"]) == (8, resident, 1), p
    assert sms - 4 * p["clusters"] < ENC_OVERLAP_MIN_SMS
    assert [q["overlap"] for q in plan] == [False, False], plan


# ---- claim order ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("bidir", [True, False], ids=["two_directions", "forward_only"])
def test_claim_order(bidir, monkeypatch):
    """bench.NET's encoder at B = 64, T = 1000: claim c beside the scan takes m-tile stream_m_tile(c // tiles_n, mid,
    tiles_m) (helpers.check_overlap_claim_order), with mid the m-tile of the frame that becomes final first: where the
    two directions meet, or frame 0 with one direction, so that a forward-only scan's claims ascend."""
    _torch()
    M = O if bidir else U
    cfg = M.make_config(**WSJ)
    rec = make_recognizer(cfg, M.init_params(cfg, seed=3, scale=10.0), bidir=bidir)
    x, m, _, _ = O.synthetic_batch(cfg, B=64, T=1000, seed=4)
    rec.encode(x, m)
    plan = rec.encoder_plan()
    assert [p["overlap"] for p in plan] == [False, True, True, True], plan
    ndir = 2 if bidir else 1
    check_overlap_claims(rec, plan, 64, cfg["subsample"], ndir)
    got = check_overlap_claim_order(rec, plan, 64, cfg["subsample"], cfg["dims_bidir"], ndir)
    print("layer: (mid, tiles beside) %s; tiles beside / all %s" % (
        got, [(p["tiles_beside"], p["tiles_beside"] + p["tiles_after"]) for p in plan[1:]]))
    assert got, plan
    if not bidir:
        assert all(mid == 0 for mid, _ in got.values()), got
