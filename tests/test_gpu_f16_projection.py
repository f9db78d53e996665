"""The fp16 head/tail operands of the projection GEMM (csrc/gemm_tc.cu: gemm_tc_kernel<true>) on the GPU, beyond what
test_gpu_encoder.py covers: which operand kind each projection of the benchmarked network runs, rows of extreme
magnitude against float64, and a training step whose forward projections take fp16 operands."""
import numpy as np
import pytest

from helpers import O, PYRAMID, WSJ, check_grads, f32, make_recognizer

pytestmark = pytest.mark.gpu

ATT = "/recognizer/generator/att_trans/conv_att"
GEMM_TOL = 5e-5          # per element, over sum_k |a_k w_k| + |b| (test_gpu_encoder.py)


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def test_operand_kind_at_the_benchmarked_widths():
    """40 features: layer 0 stays on 3xTF32 with its contraction padded to 64; layers 1-3 (K = 512) and the preprocess
    (E = 512) run on fp16 operands, unpadded."""
    _torch()
    cfg = O.make_config(**WSJ)
    rec = make_recognizer(cfg, O.init_params(cfg, seed=2, scale=10.0))
    x, m, _, _ = O.synthetic_batch(cfg, B=3, T=24, seed=2)
    att, _ = rec.encode(x, m)
    plan = rec.encoder_plan()
    assert [(p["proj"], p["kpad"], p["operands"]) for p in plan] == \
        [("tc", 64, "tf32x3")] + [("tc", 512, "f16x3")] * 3, plan
    rec.preprocess(att)
    assert rec.preprocess_plan() == {"proj": "tc", "kpad": 512}
    assert rec._encoder_plan_row(-1)["operands"] == "f16x3"


def test_no_tc_gemm_reports_no_operands(monkeypatch):
    _torch()
    monkeypatch.setenv("LVSR_NO_TC_GEMM", "1")
    cfg = O.make_config(**PYRAMID)
    rec = make_recognizer(cfg, O.init_params(cfg, seed=3, scale=10.0))
    x, m, _, _ = O.synthetic_batch(cfg, B=2, T=16, seed=3)
    rec.encode(x, m)
    assert [(p["proj"], p["operands"]) for p in rec.encoder_plan()] == [("ffma", None)] * 3


@pytest.mark.parametrize("E", [256, 512])
def test_rows_of_extreme_magnitude_against_float64(E):
    """The projection of a layer >= 1 (K = E, a multiple of 64) on rows that are all zero, near 1e-30 and near 1e30,
    next to ordinary rows, against float64.  The preprocess runs the same projection_gemm call on inputs the test
    picks (an encoder layer's input is a BiGRU output, bounded by 1).  Zero rows must give exactly the bias; the bias
    is zero for the tiny and huge rows' bound, so their error is measured over sum_k |a_k w_k| alone."""
    torch = _torch()
    M = 512
    cfg = O.make_config(**dict(PYRAMID, dims_bidir=[128, E // 2], subsample=[1, 1], dim_matcher=M))
    rng = np.random.RandomState(E)
    rows = 300
    A = rng.normal(size=(rows, E))
    A[0:37] = 0.0
    A[37:110] *= 1e-30
    A[110:190] *= 1e30
    A[190:200] *= 2.0 ** rng.randint(-20, 21, size=E)[None, :]
    W = rng.normal(size=(E, M)) * 0.05
    A, W = f32(A), f32(W)
    for b in (np.zeros(M), f32(rng.normal(size=M))):
        params = O.init_params(cfg, seed=4, scale=10.0)
        params[ATT + "/preprocess.W"], params[ATT + "/preprocess.b"] = W, b
        rec = make_recognizer(cfg, params)
        got = rec.preprocess(torch.tensor(A[:, None, :], dtype=torch.float32, device=rec.device))[:, 0]
        got = got.cpu().numpy().astype(np.float64)
        assert rec._encoder_plan_row(-1)["operands"] == "f16x3"
        assert np.isfinite(got).all()
        assert np.array_equal(got[:37], np.broadcast_to(b, (37, M)))
        want = A @ W + b
        scale = np.abs(A) @ np.abs(W) + np.abs(b)
        err = np.abs(got[37:] - want[37:]) / scale[37:]
        worst = {"1e-30": err[:73].max(), "1e30": err[73:153].max(), "spread": err[153:163].max(), "normal": err[163:].max()}
        print("E=%d bias=%s:" % (E, "yes" if b.any() else "no"), {k: "%.2e" % v for k, v in worst.items()})
        assert max(worst.values()) < GEMM_TOL, worst


def test_training_step_with_f16_forward_projections():
    """PYRAMID with [128, 128, 128]: layers 1 and 2 (K = 256) and the preprocess (E = 256) project on fp16 operands in
    the training forward; the gradients against the float64 oracle (check_grads, the bar of test_gpu_train.py)."""
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = {k: f32(v) for k, v in O.init_params(cfg, seed=11, scale=10.0).items()}
    x, m, labels, lm = O.synthetic_batch(cfg, B=5, T=40, seed=31)
    _, rec = check_grads(cfg, params, (f32(x), m, labels, lm))
    plan = rec.encoder_plan()
    assert [p["operands"] for p in plan] == ["tf32x3", "f16x3", "f16x3"], plan
    assert all(p["tape"] for p in plan) and rec._encoder_plan_row(-1)["operands"] == "f16x3"
