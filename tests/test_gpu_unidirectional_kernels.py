"""The forward-only encoder's kernels (net.bidir: False: bigru_kernel, bigru_mma_kernel and bigru_bwd_kernel with
NDIR = 1, fork projections of N = 3 D columns over K = D of the layer below) at the kernels, batches, widths and
contractions the bidirectional ones are tested at in test_gpu_encoder.py, test_gpu_bigru_rows.py, test_gpu_edges.py and
test_gpu_encoder_widths.py, against the float64 oracle of tests/unidirectional_oracle.py.  Every case reads back the
path it ran from encoder_plan() / preprocess_plan():

* the scan kernel matrix (FFMA at 128 and 256, tensor cores with 4- and 8-row clusters) on 1, 3 and 33 rows and the
  smallest batch that needs two waves of clusters with one direction, rb (resident + 1); one gradient case per kernel,
  which runs each taped variant (bigru_mma_kernel<256, 1, true, 8> only when 8-row clusters are forced);
* 8-row, 4-row and FFMA scans of a 4 x 256 forward-only encoder at 64 x 200 against each other; recurrent weights
  beyond the fp16 range on the tensor-core scan;
* gradients at D = 64, 128, 384 and 512, at T B = 2079 rows (tensor-core weight gradients, a padded contraction) with
  and without LVSR_NO_TC_GEMM, D = 512 at B = 64 (a reverse-time scan of more than one wave), and the input gradient of
  the layer above a 128-wide one;
* the fp16 projection over 1, 3, 5 and 7 64-wide k-blocks (K = 64, 192, 320, 448, which only a forward-only layer
  gives): the GEMM alone through attention.preprocess, and the fork projection of the layer above;
* a bottom MLP under a forward-only layer: layer 0's input gradient contracts over 3 D into the bottom.

Bars are the bidirectional files' (named at each test).  Worst errors measured on an H100 80GB HBM3 (700 W power
limit), which holds 30 clusters of the tensor-core scan: scans 5.1e-6 per element (SCAN_TOL 2.5e-5); RB 8 against RB 4
7.1e-7 and against FFMA 9.2e-7 (5e-6, 1e-5); weights beyond fp16 1.6e-6 (1e-4); the projection GEMM 1.9e-6 (GEMM_TOL
5e-5); the stacks above an odd-K layer 1.5e-5 ([448, 512]; STACK_TOL 4e-4); gradients 1.7e-5 of a parameter's largest
entry ([128, 512]; 1e-4).  The file runs in about 20 s."""
import numpy as np
import pytest

import bottom_oracle as BO
import unidirectional_oracle as U
from helpers import O, PYRAMID, SMALL, bottom_params, bottom_recognizer, check_unidirectional_grads, elementwise_err
from helpers import f32, make_recognizer, package, rel_err
from test_gpu_bottom import _check_grads as _check_bottom_grads, _grads as _bottom_grads
from test_gpu_encoder import ATT, GEMM_TOL, ROWS, SCAN_TOL, STACK_TOL, _gemm_operands

pytestmark = pytest.mark.gpu

KEYS = ("costs", "weights", "energies", "states", "weighted_averages")


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _f32_params(params):
    return {k: f32(v) for k, v in params.items()}


def _rec(cfg, params):
    return make_recognizer(cfg, params, bidir=False)


def _compare_encoder(cfg, params, x, m):
    """The forward-only encoder output per element (elementwise_err) and its mask exactly; (recognizer, error)."""
    params = _f32_params(params)
    x = f32(x)
    rec = _rec(cfg, params)
    att, attm = rec.encode(x, m)
    want, wmask = U.encoder(cfg, params, x, m)
    assert np.array_equal(attm.cpu().numpy(), wmask.astype(np.float32))
    return rec, elementwise_err(att.cpu().numpy(), want)


def _scan_case(cfg, params, B, T, seed, one_frame):
    x, m, _, _ = O.synthetic_batch(cfg, B=B, T=T, seed=seed, min_frac=0.3)
    if one_frame:
        m[:, 0] = np.arange(T) < 1
        x *= m[:, :, None]
    return _compare_encoder(cfg, params, x, m)


def _grads(net, B, T, seed, arch=PYRAMID):
    _torch()
    cfg = U.make_config(**dict(arch, **net))
    params = _f32_params(U.init_params(cfg, seed=seed, scale=10.0))
    x, m, labels, lm = O.synthetic_batch(cfg, B=B, T=T, seed=seed + 20)
    rec = check_unidirectional_grads(cfg, params, (f32(x), m, labels, lm))
    return rec.encoder_plan()


# ---- the scan kernel matrix --------------------------------------------------------------------------------------------

KERNELS = {                       # name -> (width, environment, kernel, rows per cluster, CTAs per cluster)
    "ffma128": (128, {}, "ffma", 4, 4),
    "ffma256": (256, {"LVSR_BIGRU_MMA": "0"}, "ffma", 4, 8),
    "mma_rb4": (256, {"LVSR_BIGRU_MMA": "1", "LVSR_BIGRU_RB": "4"}, "mma", 4, 4),
    "mma_rb8": (256, {"LVSR_BIGRU_MMA": "1", "LVSR_BIGRU_RB": "8"}, "mma", 8, 4),
}


@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_scan_kernel_matrix(kernel, monkeypatch):
    """test_gpu_encoder.py::test_bigru_kernel_matrix with one direction: 1 row, 3 rows (a partial row group), 33 rows
    and rb (resident + 1) rows, the smallest batch whose ceil(B / rb) clusters need two waves; every batch of three or
    more rows holds a one-frame utterance.  Bar SCAN_TOL per element."""
    _torch()
    D, env, name, rb, cs = KERNELS[kernel]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    cfg = U.make_config(**dict(SMALL, dims_bidir=[D]))
    params = U.init_params(cfg, seed=D, scale=10.0)
    T = 11
    rec, err = _scan_case(cfg, params, 1, T, seed=1, one_frame=False)
    resident = rec.encoder_plan()[0]["resident"]
    assert resident > 0
    two_waves = rb * (resident + 1)
    for B in (1, 3, 33, two_waves):
        if B > 1:
            rec, err = _scan_case(cfg, params, B, T, seed=B, one_frame=True)
        plan = rec.encoder_plan()[0]
        clusters = -(-B // rb)
        print("%s B=%d: %.2e" % (kernel, B, err), plan)
        assert (plan["bigru"], plan["rb"], plan["cs"], plan["tape"], plan["T"]) == (name, rb, cs, False, T), plan
        assert plan["clusters"] == clusters and plan["resident"] == resident, plan
        assert plan["waves"] == -(-clusters // resident), plan
        assert plan["waves"] == (2 if B == two_waves else 1), plan
        assert err < SCAN_TOL, (B, err)


# (B, T) of each kernel's gradient case: 8-row clusters at 33 rows leave the last cluster one row
KERNEL_GRADS = {"ffma128": (5, 24), "ffma256": (5, 24), "mma_rb4": (33, 20), "mma_rb8": (33, 20)}


@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_scan_kernel_gradients(kernel, monkeypatch):
    """The training forward of each scan kernel (its tape variant: bigru_kernel<D, CS, 1, TAPE>, and
    bigru_mma_kernel<256, 1, true, RB> at RB 4 and 8, the latter never planned at B <= 64) and the reverse-time scan of
    D / 32 CTAs, against the gradient oracle at check_grads' bar."""
    D, env, name, rb, cs = KERNELS[kernel]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    B, T = KERNEL_GRADS[kernel]
    plan = _grads(dict(dims_bidir=[D], subsample=[1]), B=B, T=T, seed=D + rb)
    p = plan[0]
    print(kernel, p)
    assert (p["bigru"], p["rb"], p["cs"], p["tape"], p["bwd_cs"]) == (name, rb, cs, True, D // 32), p
    assert p["clusters"] == -(-B // rb), p


# ---- row counts and fp16 range ----------------------------------------------------------------------------------------

def test_eight_row_clusters_agree_with_four_row_clusters(monkeypatch):
    """A forward-only 4 x 256 encoder at B = 64, T = 200 under RB 8, RB 4 and the FFMA kernel: the bars of
    test_gpu_bigru_rows.py (5e-6 of the output's largest magnitude between RB 4 and RB 8, 1e-5 against FFMA)."""
    torch = _torch()
    cfg = U.make_config(**dict(PYRAMID, dims_bidir=[256] * 4, subsample=[1, 1, 2, 2]))
    params = U.init_params(cfg, seed=9, scale=10.0)
    x, m, _, _ = O.synthetic_batch(cfg, B=64, T=200, seed=77, dtype=np.float32)
    rec = _rec(cfg, params)
    monkeypatch.setenv("LVSR_BIGRU_MMA", "0")
    ffma = rec.encode(x, m)[0].clone()
    assert [p["bigru"] for p in rec.encoder_plan()] == ["ffma"] * 4
    monkeypatch.setenv("LVSR_BIGRU_MMA", "1")
    got = {}
    for rb in (4, 8):
        monkeypatch.setenv("LVSR_BIGRU_RB", str(rb))
        got[rb] = rec.encode(x, m)[0].clone()
        assert bool(torch.isfinite(got[rb]).all()), rb
        plan = rec.encoder_plan()
        assert [(p["bigru"], p["rb"], p["clusters"]) for p in plan] == [("mma", rb, 64 // rb)] * 4, plan
    scale = float(ffma.abs().max())
    d48 = float((got[8] - got[4]).abs().max()) / scale
    d4f, d8f = (float((got[rb] - ffma).abs().max()) / scale for rb in (4, 8))
    print("rb8 vs rb4 %.2e, rb4 vs ffma %.2e, rb8 vs ffma %.2e" % (d48, d4f, d8f))
    assert d48 < 5e-6 and d4f < 1e-5 and d8f < 1e-5, (d48, d4f, d8f)


def test_recurrent_weights_beyond_the_fp16_range():
    """test_gpu_edges.py's case on the forward-only tensor-core scan: recurrent weights of 1e5 and -2.5e5 (fp16
    overflows at 65504) are rescaled by a power of two per tile; the encoder output and every output of the cost to
    1e-4 of their largest magnitude."""
    _torch()
    cfg = U.make_config(**dict(PYRAMID, dims_bidir=[256, 256], subsample=[1, 2]))
    params = U.init_params(cfg, seed=6, scale=10.0)
    for name in sorted(params):
        if name.endswith("gatedrecurrent.state_to_state") or name.endswith("gatedrecurrent.state_to_gates"):
            w = np.array(params[name])
            w[3, 5] = 1.0e5
            w[17, w.shape[1] - 2] = -2.5e5
            params[name] = w
    x, m, labels, lm = O.synthetic_batch(cfg, B=4, T=24, seed=21)
    want = U.recognizer_cost(cfg, params, x, m, labels, lm, return_all=True)
    rec = _rec(cfg, params)
    att, attm = rec.encode(x, m)
    assert [p["bigru"] for p in rec.encoder_plan()] == ["mma", "mma"], rec.encoder_plan()
    o_att, o_mask = U.encoder(cfg, params, x, m)
    errs = {"encoded": rel_err(att.cpu().numpy(), o_att)}
    assert np.array_equal(attm.cpu().numpy(), o_mask.astype(np.float32))
    got = rec.cost_matrix(labels, lm, att, attm, return_all=True)
    errs.update({k: rel_err(got[k].cpu().numpy(), want[k]) for k in KEYS if k in want})
    print({k: "%.2e" % e for k, e in errs.items()})
    for k, e in errs.items():
        assert e < 1e-4, (k, e)


# ---- backward at the remaining widths -----------------------------------------------------------------------------------

BWD = {                   # name -> (widths, B, T, LVSR_NO_TC_GEMM)
    "d64": ([64], 4, 40, False),
    "d128": ([128], 4, 40, False),
    "d384": ([384], 4, 32, False),
    "d512": ([512], 4, 24, False),
    "d128_2079_rows": ([128], 33, 63, False),
    "d512_2079_rows": ([512], 33, 63, False),
    "d128_2079_rows_no_tc": ([128], 33, 63, True),
    "d512_2079_rows_no_tc": ([512], 33, 63, True),
    "d512_b64": ([512], 64, 12, False),
    "stack_128_512": ([128, 512], 33, 63, False),
}


@pytest.mark.parametrize("case", list(BWD))
def test_gradients_at_widths(case, monkeypatch):
    """Gradients at the widths test_gpu_unidirectional.py does not train, against the gradient oracle at check_grads'
    bar.  T B = 33 * 63 = 2079 rows (>= 2048, not a multiple of 32): tensor-core weight gradients over a contraction
    padded to 2080 at 128 and 512, FFMA tiles under LVSR_NO_TC_GEMM=1.  d512_b64: the reverse-time scan of D = 512
    runs clusters of 16 CTAs (D / 32) at one CTA per SM (bwd_min_blocks), ceil(64 / 4) = 16 of them with one direction:
    256 CTAs, more than one wave on 132 SMs.  stack_128_512: layer 1's input gradient dPre W^T contracts over
    3 * 512 = 1536 columns into the 128-wide layer below, on tensor cores."""
    dims, B, T, no_tc = BWD[case]
    if no_tc:
        monkeypatch.setenv("LVSR_NO_TC_GEMM", "1")
    plan = _grads(dict(dims_bidir=dims, subsample=[1] * len(dims)), B=B, T=T, seed=len(case) + dims[-1])
    print(case, [(p["bwd_cs"], p["wgrad"], p["wgrad_kpad"], p["dx"], p["T"]) for p in plan])
    for l, p in enumerate(plan):
        assert p["bwd_cs"] == dims[l] // 32 and p["tape"] and p["T"] == T, (l, p)
        tc = not no_tc and T * B >= 2048 and dims[l] % 128 == 0
        assert (p["wgrad"], p["wgrad_kpad"]) == (("tc", -(-T * B // 32) * 32) if tc else ("ffma", 0)), (l, p)
    assert plan[0]["dx"] is None
    if B * T == 2079 and not no_tc:
        assert plan[-1]["wgrad_kpad"] == 2080 and plan[-1]["wgrad_splits"] >= 2, plan
    if case == "d512_b64":
        assert plan[0]["bwd_cs"] * -(-B // 4) == 256, plan
    if case == "stack_128_512":
        assert plan[1]["dx"] == "tc", plan


# ---- fp16 projections over an odd number of 64-wide k-blocks -----------------------------------------------------------

ODD_K = [64, 192, 320, 448]      # 1, 3, 5, 7 k-blocks of TC_BK_F16 = 64


@pytest.mark.parametrize("E", ODD_K)
def test_projection_gemm_at_odd_k_blocks(E):
    """attention.preprocess (the fork projection's GEMM) at K = E = dims[-1] of a forward-only encoder, on fp16
    head/tail operands, M = 256 columns: 1, 127, 128, 129 and 4097 rows, normal inputs and columns spanning
    2^-20..2^20.  Per element over sum_k |a_k w_k| + |b|, bar GEMM_TOL["tc"]."""
    torch = _torch()
    M = 256
    cfg = U.make_config(**dict(SMALL, dims_bidir=[E], dim_matcher=M))
    worst = {}
    for ri, regime in enumerate(("normal", "spread")):
        A, W, b = _gemm_operands(regime, max(ROWS), E, M, seed=E + M + ri)
        params = U.init_params(cfg, seed=3, scale=10.0)
        params[ATT + "/preprocess.W"], params[ATT + "/preprocess.b"] = W, b
        rec = _rec(cfg, params)
        for rows in ROWS:
            a = A[:rows]
            got = rec.preprocess(torch.tensor(a[:, None, :], dtype=torch.float32, device=rec.device))[:, 0]
            got = got.cpu().numpy().astype(np.float64)
            assert rec.preprocess_plan() == {"proj": "tc", "kpad": E}, rec.preprocess_plan()
            assert rec._encoder_plan_row(-1)["operands"] == "f16x3"
            want = a @ W + b
            scale = np.abs(a) @ np.abs(W) + np.abs(b)
            worst[regime] = max(worst.get(regime, 0.0), float((np.abs(got - want) / scale).max()))
    print("projection K=%d:" % E, {k: "%.2e" % v for k, v in worst.items()})
    for regime, err in worst.items():
        assert err < GEMM_TOL["tc"], (regime, err)


@pytest.mark.parametrize("dims", [[64, 128], [192, 256], [320, 384], [448, 512]], ids=lambda d: "%d_%d" % tuple(d))
def test_fork_projection_above_an_odd_k_layer(dims):
    """Layer 1 projects layer 0's D0 = 64 .. 448 features onto 3 D1 columns (a multiple of 128) on fp16 operands,
    unpadded, while layer 0 (3 D0 not a multiple of 128) projects on FFMA; 5 ragged rows with a one-frame utterance.
    The encoder output per element, bar STACK_TOL."""
    _torch()
    cfg = U.make_config(**dict(SMALL, dims_bidir=dims, subsample=[1, 1]))
    params = U.init_params(cfg, seed=dims[0], scale=10.0)
    rec, err = _scan_case(cfg, params, 5, 21, seed=dims[1], one_frame=True)
    plan = rec.encoder_plan()
    print(dims, "%.2e" % err, [(p["proj"], p["kpad"], p["operands"], p["bigru"]) for p in plan])
    assert plan[0]["proj"] == "ffma", plan
    assert (plan[1]["proj"], plan[1]["kpad"], plan[1]["operands"]) == ("tc", dims[0], "f16x3"), plan
    assert err < STACK_TOL, err


# ---- a bottom MLP under a forward-only layer ---------------------------------------------------------------------------

BOTTOM_CASES = {                # name -> (activation, B, T, LVSR_NO_TC_GEMM)
    "tanh_2079_rows_tc": ("tanh", 33, 63, False),
    "relu_ffma": ("relu", 4, 40, True),
}


@pytest.mark.parametrize("case", list(BOTTOM_CASES))
def test_bottom_mlp_gradients(case, monkeypatch):
    """bottom.dims [256, 128] under a forward-only [256] layer: layer 0's input gradient dPre W^T contracts over
    3 D = 768 columns into the bottom's 128 outputs, on tensor cores at T B = 33 * 63 = 2079 rows (Tanh: over that many
    rows some Rectifier pre-activation always lies within float32 error of its kink, as test_gpu_bottom.py's 2048-row
    cases find), and on FFMA tiles under LVSR_NO_TC_GEMM=1 with a Rectifier bottom.  Against bottom_oracle composed with
    unidirectional_oracle (pinned on the CPU by tests/test_bench_uni_golden_cpu.py), at check_grads' bar."""
    _torch()
    activation, B, T, no_tc = BOTTOM_CASES[case]
    if no_tc:
        monkeypatch.setenv("LVSR_NO_TC_GEMM", "1")
    cfg = BO.make_config(U.make_config(**dict(SMALL, dims_bidir=[256])), [256, 128], activation)
    params = bottom_params(cfg, seed=23)
    batch = O.synthetic_batch(cfg, B=B, T=T, seed=24)
    assert not BO.kinks(cfg, params, batch[0], batch[1])
    rec = bottom_recognizer(cfg, params)
    cost, grads = _bottom_grads(rec, batch)
    _check_bottom_grads(cfg, params, batch, cost, grads)
    p = rec.encoder_plan()[0]
    print(p)
    assert p["dx"] == ("ffma" if no_tc else "tc") and p["bwd_cs"] == 8 and p["tape"], p
    assert not any("/bidir0/" in k for k in grads)
