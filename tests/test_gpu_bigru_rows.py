"""8-row clusters of the tensor-core BiGRU (csrc/bigru.cu: bigru_mma_kernel<256, TAPE, 8>).  bigru_layer picks them
when they need fewer waves than 4-row clusters (the metric batch, B = 64); LVSR_BIGRU_RB=4|8 forces either variant so
both run here on any part.  Same oracle bars as the 4-row kernel's tests in test_gpu_edges.py."""
import numpy as np
import pytest

from helpers import O, PYRAMID, WSJ, check_grads, make_recognizer, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4
KEYS = ("costs", "weights", "energies", "states", "weighted_averages")
ENC256 = dict(PYRAMID, dims_bidir=[256, 256], subsample=[1, 2])
WSJ_ENC = dict(PYRAMID, dims_bidir=[256, 256, 256, 256], subsample=[1, 1, 2, 2])


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def test_eight_row_clusters_agree_with_four_row_clusters(monkeypatch):
    """Both row counts compute the same three products per k-step and differ only in the order of the fp32 accumulation
    (RB = 4 sums even and odd k-steps in separate chains).  After four layers of 200 steps that moves the encoder output
    by about 2e-6 of its largest magnitude: as much as any two fp32 orders differ here, e.g. RB = 4 against the FFMA
    kernel.  Hence 5e-6 between the two; each agrees with the FFMA kernel to 1e-5 (the bar of
    test_tensor_core_bigru_agrees_with_the_fp32_kernel)."""
    torch = _torch()
    cfg = O.make_config(**WSJ_ENC)
    params = O.init_params(cfg, seed=9, scale=10.0)
    x, m, _, _ = O.synthetic_batch(cfg, B=64, T=200, seed=77, dtype=np.float32)
    rec = make_recognizer(cfg, params)
    monkeypatch.setenv("LVSR_BIGRU_MMA", "0")
    ffma = rec.encode(x, m)[0].clone()
    assert [p["bigru"] for p in rec.encoder_plan()] == ["ffma"] * 4
    monkeypatch.setenv("LVSR_BIGRU_MMA", "1")
    got = {}
    for rb in (4, 8):
        monkeypatch.setenv("LVSR_BIGRU_RB", str(rb))
        got[rb] = rec.encode(x, m)[0].clone()
        assert bool(torch.isfinite(got[rb]).all()), rb
        assert [(p["bigru"], p["rb"]) for p in rec.encoder_plan()] == [("mma", rb)] * 4
    scale = float(ffma.abs().max())
    d48 = float((got[8] - got[4]).abs().max()) / scale
    d4f, d8f = (float((got[rb] - ffma).abs().max()) / scale for rb in (4, 8))
    print("rb8 vs rb4 %.2e, rb4 vs ffma %.2e, rb8 vs ffma %.2e" % (d48, d4f, d8f))
    assert d48 < 5e-6 and d4f < 1e-5 and d8f < 1e-5, (d48, d4f, d8f)


def _compare_cost(cfg, params, x, m, labels, lm):
    want = O.recognizer_cost(cfg, params, x, m, labels, lm, return_all=True)
    rec = make_recognizer(cfg, params)
    att, attm = rec.encode(x, m)
    o_att, o_mask = O.encoder(cfg, params, x, m)
    assert rel_err(att.cpu().numpy(), o_att) < TOL
    assert np.array_equal(attm.cpu().numpy(), o_mask.astype(np.float32))
    got = rec.cost_matrix(labels, lm, att, attm, return_all=True)
    for k in KEYS:
        if k in want:
            e = rel_err(got[k].cpu().numpy(), want[k])
            assert e < TOL, (k, e)


@pytest.mark.parametrize("B,T", [(1, 9), (7, 33), (9, 8), (33, 21), (70, 12), (300, 10)])
def test_eight_row_clusters_odd_shapes(B, T, monkeypatch):
    """Batches that leave the last 8-row cluster partly empty (1, 7, 9, 33, 70 rows), lengths that are not multiples of
    the subsampling, a one-frame utterance, and 300 rows = 76 clusters: more than any H100 holds at once, so the launch
    runs in waves.  Against the float64 oracle."""
    _torch()
    monkeypatch.setenv("LVSR_BIGRU_RB", "8")
    cfg = O.make_config(**ENC256)
    params = O.init_params(cfg, seed=4, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=B, T=T, seed=B * 10 + T, min_frac=0.2)
    if B >= 3:
        m[:, 0] = (np.arange(T) < 1)          # a one-frame utterance
        x *= m[:, :, None]
    _compare_cost(cfg, params, x, m, labels, lm)


def test_eight_row_clusters_training_gradients(monkeypatch):
    """The training forward (TAPE: gates, candidates and every frame of h kept for the reverse-time scan) under 8-row
    clusters at the metric batch: gradients of every parameter of the WSJ architecture against the gradient oracle."""
    _torch()
    monkeypatch.setenv("LVSR_BIGRU_RB", "8")
    cfg = O.make_config(**WSJ)
    params = O.init_params(cfg, seed=1, scale=10.0)
    batch = O.synthetic_batch(cfg, B=64, T=48, seed=3)
    check_grads(cfg, params, batch)


def test_row_count_switch_rejects_other_values(monkeypatch):
    _torch()
    monkeypatch.setenv("LVSR_BIGRU_RB", "16")
    cfg = O.make_config(**ENC256)
    rec = make_recognizer(cfg, O.init_params(cfg, seed=4, scale=10.0))
    x, m, _, _ = O.synthetic_batch(cfg, B=4, T=8, seed=1)
    with pytest.raises(Exception, match="LVSR_BIGRU_RB"):
        rec.encode(x, m)
