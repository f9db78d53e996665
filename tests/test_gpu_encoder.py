"""The encoder's kernels element by element against the float64 oracle, with the path every case ran read back from
the encoder plan report (lvsr_model_encoder_plan / SpeechRecognizer.encoder_plan):

* the projection GEMM alone (attention.preprocess runs exactly the fork projection's GEMM on inputs the test picks):
  the 3xTF32 tensor-core kernel (csrc/gemm_tc.cu) and the FFMA tile kernel (csrc/gemm.cu) at partial and single M tiles,
  on normal inputs, on coherent positive inputs whose tf32 low parts are near their largest (where a dropped cross
  product of the split would add up) and on columns whose magnitudes span 2^-20..2^20;
* the layer-0 projection at every number of 32-float k-blocks the kernel's 3-stage ring distinguishes, and the FFMA
  fallback for feature widths that are not a multiple of 4;
* the four BiGRU scan kernels (csrc/bigru.cu: FFMA at 128 and 256, tensor-core with 4- and 8-row clusters) on partial
  row groups, a one-frame utterance and a batch that needs more than one wave of clusters, and stacks with subsampling
  remainders, a factor longer than the layer, mixed widths and LVSR_MAX_LAYERS layers;
* the training step (check_grads, the bar of test_gpu_train.py) on the tensor-core and FFMA weight gradients with a
  contraction over T*B rows that is not a multiple of 32, layers whose length is not a multiple of their subsampling
  (csrc/bigru_bwd.cu), the FFMA scan with its tape at 256 and 8-row clusters.

Inputs and parameters given to the oracle are the float32 values the kernels see (helpers.f32), so every error measured
is the kernels' own.  Bounds sit 4-10x above the worst error measured on an H100 (DESIGN §2)."""
import numpy as np
import pytest

from helpers import O, PYRAMID, SMALL, check_grads, elementwise_err, f32, make_recognizer, package

pytestmark = pytest.mark.gpu

ATT = "/recognizer/generator/att_trans/conv_att"
# per element, over sum_k |a_k w_k| + |b|.  Tensor cores: 1.2e-5 measured (coherent inputs, E = 512), while a split that
# dropped a cross product errs by about 6e-4 there; FFMA: 1.8e-6 measured
GEMM_TOL = {"tc": 5e-5, "ffma": 1e-5}
# encoder output per element (elementwise_err, floor 0.1 of the largest magnitude)
LAYER0_TOL = 8e-5        # one layer, 1 to 260 features: 1.6e-5 measured (260 features)
SCAN_TOL = 2.5e-5        # one layer, every scan kernel and batch: 5.1e-6 measured
STACK_TOL = 4e-4         # stacks of 2 to 8 layers: the error grows with depth (1.0e-4 measured at 8 layers)


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _f32_params(params):
    return {k: f32(v) for k, v in params.items()}


# ---- the projection GEMM alone ----------------------------------------------------------------------------------------

def _tf32_low_near_max(rng, shape, lo=1.0):
    """Positive float32 values in [lo, 2 lo): random top 10 mantissa bits (the tf32 part), the low 13 bits in
    [0x1C00, 0x1FFF] -- the tf32 split leaves a low part of almost one tf32 ulp in every operand."""
    top = rng.randint(0, 1 << 10, size=shape).astype(np.uint32)
    low = rng.randint(0x1C00, 0x2000, size=shape).astype(np.uint32)
    bits = (np.uint32(127) << np.uint32(23)) | (top << np.uint32(13)) | low
    return bits.view(np.float32).astype(np.float64) * lo


def _gemm_operands(regime, rows, E, M, seed):
    rng = np.random.RandomState(seed)
    if regime == "normal":
        A = rng.normal(size=(rows, E))
        W = rng.normal(size=(E, M)) * 0.1
        b = rng.normal(size=M)
    elif regime == "coherent":
        A = _tf32_low_near_max(rng, (rows, E))
        W = _tf32_low_near_max(rng, (E, M), 2.0 ** -4)
        b = _tf32_low_near_max(rng, M)
    else:                                                   # per-column magnitudes 2^-20 .. 2^20
        A = rng.normal(size=(rows, E)) * 2.0 ** rng.randint(-20, 21, size=E)[None, :]
        W = rng.normal(size=(E, M)) * 2.0 ** rng.randint(-20, 21, size=M)[None, :]
        b = rng.normal(size=M) * 2.0 ** rng.randint(-20, 21, size=M)
    return f32(A), f32(W), f32(b)


ROWS = (1, 127, 128, 129, 4097)
REGIMES = ("normal", "coherent", "spread")


@pytest.mark.parametrize("path", ["tc", "ffma"])
@pytest.mark.parametrize("M", [128, 256, 512])
@pytest.mark.parametrize("E", [256, 512])
def test_projection_gemm_against_float64(E, M, path, monkeypatch):
    """preprocess = attended . W + b on the tensor cores (3xTF32: lo.hi + hi.lo + hi.hi, DESIGN §2) and, under
    LVSR_NO_TC_GEMM=1 (read when the weights are packed), on FFMA tiles: 1, 127, 128, 129 and 4097 rows, three input
    regimes.  Each element's error is measured over sum_k |a_k w_k| + |b|: the coherent regime keeps that sum equal to
    the result, so a split that dropped one cross product would show its 2^-11 relative error there in full."""
    torch = _torch()
    if path == "ffma":
        monkeypatch.setenv("LVSR_NO_TC_GEMM", "1")
    cfg = O.make_config(**dict(SMALL, dims_bidir=[E // 2], dim_matcher=M))
    worst = {}
    for ri, regime in enumerate(REGIMES):
        A, W, b = _gemm_operands(regime, max(ROWS), E, M, seed=E + M + ri)
        params = O.init_params(cfg, seed=3, scale=10.0)
        params[ATT + "/preprocess.W"], params[ATT + "/preprocess.b"] = W, b
        rec = make_recognizer(cfg, params)
        for rows in ROWS:
            a = A[:rows]
            got = rec.preprocess(torch.tensor(a[:, None, :], dtype=torch.float32, device=rec.device))[:, 0]
            got = got.cpu().numpy().astype(np.float64)
            plan = rec.preprocess_plan()
            assert plan == ({"proj": "tc", "kpad": E} if path == "tc" else {"proj": "ffma", "kpad": 0}), plan
            want = a @ W + b
            scale = np.abs(a) @ np.abs(W) + np.abs(b)
            err = float((np.abs(got - want) / scale).max())
            worst[regime] = max(worst.get(regime, 0.0), err)
    print("projection E=%d M=%d %s:" % (E, M, path), {k: "%.2e" % v for k, v in worst.items()})
    for regime, err in worst.items():
        assert err < GEMM_TOL[path], (regime, err)


# ---- layer-0 contraction widths ---------------------------------------------------------------------------------------

def _compare_encoder(cfg, params, x, m):
    """Encoder output per element and its mask exactly; returns (recognizer, error)."""
    params = _f32_params(params)
    x = f32(x)
    rec = make_recognizer(cfg, params)
    att, attm = rec.encode(x, m)
    o_att, o_mask = O.encoder(cfg, params, x, m)
    assert np.array_equal(attm.cpu().numpy(), o_mask.astype(np.float32))
    err = elementwise_err(att.cpu().numpy(), o_att)
    return rec, err


# features -> tf32-padded contraction of the layer-0 projection (0: the FFMA kernel, K % 4 != 0)
FEATURES = {1: 0, 2: 0, 123: 0, 4: 32, 32: 32, 36: 64, 40: 64, 96: 96, 128: 128, 260: 288}


@pytest.mark.parametrize("D", [128, 256])
@pytest.mark.parametrize("F", sorted(FEATURES))
def test_layer0_contraction_widths(F, D):
    """One-layer encoders: one k-block (4, 32 features), a padded second block (36, 40), exactly the ring's three
    stages (96), one wrap of the ring (128), nine blocks after padding (260), and the FFMA kernel for widths that are
    not a multiple of 4 (1, 2, 123).  The features are scaled by sqrt(40 / F), so that the pre-activations have the same
    spread at every width and one bound fits all."""
    _torch()
    cfg = O.make_config(**dict(SMALL, num_features=F, dims_bidir=[D]))
    params = O.init_params(cfg, seed=F, scale=10.0)
    x, m, _, _ = O.synthetic_batch(cfg, B=5, T=21, seed=F + D)
    rec, err = _compare_encoder(cfg, params, x * np.sqrt(40.0 / F), m)
    plan = rec.encoder_plan()[0]
    print("F=%d D=%d: %.2e" % (F, D, err), plan)
    assert plan["proj"] == ("tc" if FEATURES[F] else "ffma") and plan["kpad"] == FEATURES[F], plan
    assert err < LAYER0_TOL, err


# ---- the BiGRU kernel matrix ------------------------------------------------------------------------------------------

KERNELS = {                       # name -> (width, environment, kernel, rows per cluster, CTAs per cluster)
    "ffma128": (128, {}, "ffma", 4, 4),
    "ffma256": (256, {"LVSR_BIGRU_MMA": "0"}, "ffma", 4, 8),
    "mma_rb4": (256, {"LVSR_BIGRU_MMA": "1", "LVSR_BIGRU_RB": "4"}, "mma", 4, 4),
    "mma_rb8": (256, {"LVSR_BIGRU_MMA": "1", "LVSR_BIGRU_RB": "8"}, "mma", 8, 4),
}


def _scan_case(cfg, params, B, T, seed, one_frame):
    x, m, _, _ = O.synthetic_batch(cfg, B=B, T=T, seed=seed, min_frac=0.3)
    if one_frame:
        m[:, 0] = np.arange(T) < 1
        x *= m[:, :, None]
    return _compare_encoder(cfg, params, x, m)


@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_bigru_kernel_matrix(kernel, monkeypatch):
    """Each scan kernel on 1 row, 3 rows (a partial row group), 33 rows and, from the occupancy answer the plan
    reports, the smallest batch that needs two waves of clusters; every batch of three or more rows holds a one-frame
    utterance."""
    _torch()
    D, env, name, rb, cs = KERNELS[kernel]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    cfg = O.make_config(**dict(SMALL, dims_bidir=[D]))
    params = O.init_params(cfg, seed=D, scale=10.0)
    T = 11
    rec, err = _scan_case(cfg, params, 1, T, seed=1, one_frame=False)
    resident = rec.encoder_plan()[0]["resident"]
    assert resident > 0
    two_waves = rb * (resident // 2 + 1)                  # 2 * ceil(B / rb) > resident clusters
    for B in (1, 3, 33, two_waves):
        if B > 1:
            rec, err = _scan_case(cfg, params, B, T, seed=B, one_frame=True)
        plan = rec.encoder_plan()[0]
        clusters = 2 * -(-B // rb)
        print("%s B=%d: %.2e" % (kernel, B, err), plan)
        assert (plan["bigru"], plan["rb"], plan["cs"], plan["tape"], plan["T"]) == (name, rb, cs, False, T), plan
        assert plan["clusters"] == clusters and plan["resident"] == resident, plan
        assert plan["waves"] == -(-clusters // resident), plan
        assert plan["waves"] == 1 if B == 1 else plan["waves"] >= 2 if B == two_waves else True, plan
        assert err < SCAN_TOL, (B, err)


STACKS = {                        # name -> (widths, subsampling, T, B)
    "remainder_1_3": ([128, 128], [1, 3], 62, 5),
    "remainder_2_2_2": ([128, 128, 128], [2, 2, 2], 61, 5),
    "factor_beyond_length": ([128, 128], [1, 4], 3, 4),
    "mixed_widths": ([128, 256, 128, 256], [1, 2, 1, 1], 30, 5),
    "max_layers": ([128, 256, 128, 128, 256, 128, 128, 128], [1, 1, 2, 1, 1, 2, 1, 1], 24, 3),
}


@pytest.mark.parametrize("stack", sorted(STACKS))
def test_encoder_stacks(stack):
    """Layers whose length is not a multiple of their subsampling (62 -> 21, 61 -> 31 -> 16 -> 8), a factor longer
    than the layer (3 frames, factor 4: one encoded frame), a width change at every layer boundary and a stack of
    LVSR_MAX_LAYERS = 8 layers; ragged masks and a one-frame utterance."""
    _torch()
    dims, sub, T, B = STACKS[stack]
    cfg = O.make_config(**dict(SMALL, dims_bidir=dims, subsample=sub))
    params = O.init_params(cfg, seed=len(dims), scale=10.0)
    rec, err = _scan_case(cfg, params, B, T, seed=T, one_frame=True)
    plan = rec.encoder_plan()
    print(stack, "%.2e" % err, [(p["T"], p["bigru"], p["proj"]) for p in plan])
    Tl = T
    for l, p in enumerate(plan):
        assert p["T"] == Tl and p["bigru"] == ("mma" if dims[l] == 256 else "ffma") and p["proj"] == "tc", (l, p)
        Tl = -(-Tl // sub[l])
    assert rec.encoded_length(T) == Tl
    assert err < STACK_TOL, err


# ---- the training step ------------------------------------------------------------------------------------------------

def _grads(net, B, T, seed):
    _torch()
    cfg = O.make_config(**dict(PYRAMID, **net))
    params = _f32_params(O.init_params(cfg, seed=seed, scale=10.0))
    x, m, labels, lm = O.synthetic_batch(cfg, B=B, T=T, seed=seed + 20)
    _, rec = check_grads(cfg, params, (f32(x), m, labels, lm))
    return rec.encoder_plan()


def _bwd(plan):
    return [(p["wgrad"], p["wgrad_kpad"], p["dx"], p["bwd_cs"]) for p in plan]


@pytest.mark.parametrize("no_tc", [False, True], ids=["tc", "no_tc"])
def test_gradients_with_a_padded_contraction_and_a_remainder(no_tc, monkeypatch):
    """B = 33, T = 63: T*B = 2079 rows, so layers 0 and 1 take the tensor-core weight gradients with the contraction
    padded to 2080 and a short last split; layer 1 (63 frames, factor 2) leaves its last frame without an output
    gradient of its own; 33 rows leave a partial 4-row group in the backward kernel.  Under LVSR_NO_TC_GEMM=1 every
    product runs on FFMA tiles."""
    if no_tc:
        monkeypatch.setenv("LVSR_NO_TC_GEMM", "1")
    plan = _grads({}, B=33, T=63, seed=5)
    if no_tc:
        assert _bwd(plan) == [("ffma", 0, None, 4), ("ffma", 0, "ffma", 4), ("ffma", 0, "ffma", 4)], plan
        assert [p["proj"] for p in plan] == ["ffma"] * 3
    else:
        assert _bwd(plan) == [("tc", 2080, None, 4), ("tc", 2080, "tc", 4), ("ffma", 0, "tc", 4)], plan
        assert plan[0]["wgrad_splits"] >= 2 and [p["proj"] for p in plan] == ["tc"] * 3
    assert [p["T"] for p in plan] == [63, 63, 32] and all(p["tape"] for p in plan)


@pytest.mark.parametrize("no_tc", [False, True], ids=["tc", "no_tc"])
def test_gradients_256_with_a_padded_contraction_and_a_remainder(no_tc, monkeypatch):
    """The 256-wide stack [256, 256] / [1, 2] at B = 33, T = 63: the 8-CTA backward kernel on a partial row group, the
    tensor-core scan with its tape, and both weight-gradient paths with 2079 rows."""
    if no_tc:
        monkeypatch.setenv("LVSR_NO_TC_GEMM", "1")
    plan = _grads(dict(dims_bidir=[256, 256], subsample=[1, 2]), B=33, T=63, seed=6)
    if no_tc:
        assert _bwd(plan) == [("ffma", 0, None, 8), ("ffma", 0, "ffma", 8)], plan
    else:
        assert _bwd(plan) == [("tc", 2080, None, 8), ("tc", 2080, "tc", 8)], plan
    assert all(p["bigru"] == "mma" and p["tape"] for p in plan), plan


def test_gradients_ffma_scan_with_tape_at_256(monkeypatch):
    """LVSR_BIGRU_MMA=0 at hidden size 256: the training forward runs the FFMA kernel with its tape stores
    (bigru_kernel<256, 8, 8, TAPE = true>)."""
    monkeypatch.setenv("LVSR_BIGRU_MMA", "0")
    plan = _grads(dict(dims_bidir=[256], subsample=[1]), B=5, T=24, seed=7)
    assert (plan[0]["bigru"], plan[0]["cs"], plan[0]["tape"], plan[0]["bwd_cs"]) == ("ffma", 8, True, 8), plan


def test_gradients_eight_row_clusters_at_33_rows(monkeypatch):
    """LVSR_BIGRU_RB=8 at B = 33: the last 8-row cluster of the tensor-core scan holds one row."""
    monkeypatch.setenv("LVSR_BIGRU_RB", "8")
    plan = _grads(dict(dims_bidir=[256], subsample=[1]), B=33, T=20, seed=8)
    assert (plan[0]["bigru"], plan[0]["rb"], plan[0]["clusters"], plan[0]["tape"]) == ("mma", 8, 10, True), plan


def test_gradients_36_features_above_2048_rows():
    """36 features at 2079 rows: the first weight-gradient product has 36 output rows (a partial M tile) and a padded
    contraction, and the forward projection pads 36 to 64."""
    plan = _grads(dict(num_features=36, dims_bidir=[128], subsample=[1]), B=33, T=63, seed=9)
    assert (plan[0]["proj"], plan[0]["kpad"]) == ("tc", 64), plan
    assert _bwd(plan) == [("tc", 2080, None, 4)], plan


def test_gradients_small_batch_with_subsampling_remainders():
    """[1, 3, 2] at T = 47: 47 -> 16 -> 8 frames; layer 1 (47 frames, factor 3) leaves two trailing frames without an
    output gradient of their own."""
    plan = _grads(dict(subsample=[1, 3, 2]), B=4, T=47, seed=10)
    assert [p["T"] for p in plan] == [47, 47, 16], plan
    assert _bwd(plan) == [("ffma", 0, None, 4), ("ffma", 0, "tc", 4), ("ffma", 0, "tc", 4)], plan


def test_plan_report_before_and_after_training():
    """An inference forward reports no tape and leaves the backward slots at zero; layer -1 is the last preprocess;
    layers outside the stack are refused.  ABI 104."""
    _torch()
    pkg = package()
    assert pkg._lib.load().lvsr_version() == 104
    cfg = O.make_config(**SMALL)
    rec = make_recognizer(cfg, O.init_params(cfg, seed=1, scale=10.0))
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=16, seed=1)
    att, attm = rec.encode(x, m)
    plan = rec.encoder_plan()
    assert len(plan) == 1 and plan[0]["tape"] is False and plan[0]["T"] == 16 and plan[0]["kpad"] == 64, plan
    assert _bwd(plan) == [(None, 0, None, 0)]
    rec.preprocess(att)
    assert rec.preprocess_plan() == {"proj": "tc", "kpad": 256}
    import ctypes as C
    out = (C.c_int32 * 16)()
    assert pkg._lib.load().lvsr_model_encoder_plan(rec._require_ready(), 1, out) != 0
