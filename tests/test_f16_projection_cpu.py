"""Numerics of the fp16 operands of the projection GEMM (csrc/gemm_tc.cu: split_rows_f16_kernel,
transpose_split_f16_kernel, the epilogue of gemm_tc_kernel<true>) restated in numpy, and the compiled form of that kernel.

Every row of A (every column of W) is scaled by 2^e, e = 140 - the biased exponent of its largest magnitude (clamped to
127; 0 for an all-zero vector), which puts that magnitude into [2^13, 2^14).  Then y = x 2^e = head + tail with
head = fp16(y), tail = fp16(y - head); three products are accumulated and the epilogue computes
ldexp(acc, -(e_row + e_col)) + bias.  The claim in DESIGN.md section 2: head + tail is within 2^-22 of |y|, or 2^-25
absolute where the tail is an fp16 subnormal, and the unscaling is exact."""
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "attention-lvcsr_b200", "csrc")


def range_exponent(max_abs):
    """mirror of f16_range_exponent() in gemm_tc.cu"""
    max_abs = np.asarray(max_abs, dtype=np.float32)
    biased = ((max_abs.view(np.uint32) >> np.uint32(23)) & np.uint32(0xFF)).astype(np.int64)
    return np.where(max_abs == 0, 0, np.minimum(140 - biased, 127))


def split_rows(x):
    """[M, K] float32 -> (head, tail) float16 [M, K] and the row exponents [M]"""
    x = np.asarray(x, dtype=np.float32)
    e = range_exponent(np.abs(x).max(axis=1))
    y = (x * np.ldexp(np.float32(1), e)[:, None].astype(np.float32)).astype(np.float32)
    head = y.astype(np.float16)
    tail = (y - head.astype(np.float32)).astype(np.float16)
    return head, tail, e


def split_gemm(a, w, bias):
    """a [M, K] . w [K, N] + bias the way the kernel combines the parts (products and sums in float64: the tensor core's
    fp32 accumulation adds its own 2^-24 per term, which is not what is under test)"""
    ah, at, ea = split_rows(a)
    wh, wt, ew = split_rows(np.asarray(w, np.float32).T)
    ah, at, wh, wt = (v.astype(np.float64) for v in (ah, at, wh, wt))
    acc = at @ wh.T + ah @ wt.T + ah @ wh.T
    return np.ldexp(acc, -(ea[:, None] + ew[None, :])) + bias


def _rows(rng):
    K = 512
    return np.concatenate([
        rng.normal(size=(8, K)),
        rng.uniform(-1, 1, (8, K)),
        rng.normal(size=(8, K)) * 2.0 ** rng.randint(-20, 21, size=K)[None, :],   # the spread regime's columns
        rng.normal(size=(4, K)) * 1e-30,
        rng.normal(size=(4, K)) * 1e30,
    ]).astype(np.float32)


def test_exponent_puts_the_largest_magnitude_into_2_pow_13_14():
    rng = np.random.RandomState(0)
    x = _rows(rng)
    _, _, e = split_rows(x)
    top = np.abs(x).max(axis=1).astype(np.float64) * 2.0 ** e
    assert ((top >= 2.0 ** 13) & (top < 2.0 ** 14)).all(), top
    assert range_exponent(np.float32(8192.0)) == 0 and range_exponent(np.float32(16383.0)) == 0
    assert range_exponent(np.float32(16384.0)) == -1 and range_exponent(np.float32(1.0)) == 13
    assert range_exponent(np.float32(3.4e38)) == -114                   # every finite row scales down exactly
    assert range_exponent(np.float32(1e-40)) == 127                     # subnormal rows: 2^127 is the largest scale


def test_head_plus_tail_within_2_pow_minus_22_or_2_pow_minus_25():
    rng = np.random.RandomState(1)
    x = _rows(rng)
    head, tail, e = split_rows(x)
    assert np.isfinite(head.astype(np.float32)).all() and np.isfinite(tail.astype(np.float32)).all()
    y = x.astype(np.float64) * 2.0 ** e[:, None]                        # exact: powers of two
    back = head.astype(np.float64) + tail.astype(np.float64)
    assert (np.abs(back - y) <= np.maximum(2.0 ** -22 * np.abs(y), 2.0 ** -25)).all()
    # 2^-25 absolute is 2^-38 of the row maximum
    assert (np.abs(back - y).max(axis=1) / np.abs(y).max(axis=1) <= 2.0 ** -22).all()


def test_all_zero_rows_get_exponent_0_and_give_the_bias():
    x = np.zeros((3, 64), np.float32)
    head, tail, e = split_rows(x)
    assert (e == 0).all() and not head.any() and not tail.any()
    rng = np.random.RandomState(2)
    w = rng.normal(size=(64, 128)).astype(np.float32)
    b = rng.normal(size=128)
    assert np.array_equal(split_gemm(x, w, b), np.broadcast_to(b, (3, 128)))


@pytest.mark.parametrize("magnitude", [1e-30, 1.0, 1e30])
def test_split_product_matches_float64_at_every_row_magnitude(magnitude):
    rng = np.random.RandomState(3)
    K, N = 512, 256
    a = (rng.normal(size=(16, K)) * magnitude).astype(np.float32)
    w = (rng.normal(size=(K, N)) * 0.05 * 2.0 ** rng.randint(-20, 21, size=N)[None, :]).astype(np.float32)
    a64, w64 = a.astype(np.float64), w.astype(np.float64)
    exact = a64 @ w64
    bound = np.abs(a64) @ np.abs(w64)
    got = split_gemm(a, w, 0.0)
    assert (np.abs(got - exact) / bound).max() < 2.0 ** -20


def test_epilogue_unscale_round_trips_exactly():
    """ldexp(acc, -(e_row + e_col)) undoes the two scalings exactly whenever the result is a normal float32, including
    exponent sums beyond the range of one float32 power of two"""
    rng = np.random.RandomState(4)
    v = rng.normal(size=64).astype(np.float32)
    for er, ec in ((0, 0), (13, -40), (113, 113), (-100, -14), (127, 127), (-114, 100)):
        with np.errstate(over="ignore"):
            acc = (v.astype(np.float64) * 2.0 ** (er + ec)).astype(np.float32)
        back = np.ldexp(acc.astype(np.float64), -(er + ec)).astype(np.float32)
        if np.isfinite(acc).all() and (np.abs(acc[acc != 0]) >= np.finfo(np.float32).tiny).all():
            assert np.array_equal(back, v), (er, ec)


NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.fixture(scope="module")
def gemm_tc_build():
    """gemm_tc.cu compiled on its own for sm_90a: the ptxas report and the SASS of each gemm_tc_kernel instantiation"""
    if not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)):
        pytest.skip("nvcc or cuobjdump missing")
    with tempfile.TemporaryDirectory() as tmp:
        obj = os.path.join(tmp, "gemm_tc.o")
        cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
               "-I" + os.path.join(CSRC, "..", "..", "include"), "-I" + CSRC, "-c", os.path.join(CSRC, "gemm_tc.cu"),
               "-o", obj]
        ptxas = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
        sass = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name and "/*" in line:
            funcs[name].append(line)
    return ptxas, {k: "\n".join(v) for k, v in funcs.items()}


def test_f16_instantiation_runs_k16_wgmma_and_the_tf32_one_k8(gemm_tc_build):
    _, funcs = gemm_tc_build
    f16 = [v for k, v in funcs.items() if "gemm_tc_kernelILb1E" in k]
    tf32 = [v for k, v in funcs.items() if "gemm_tc_kernelILb0E" in k]
    assert len(f16) == 1 and len(tf32) == 1, sorted(funcs)
    assert re.search(r"HGMMA\.64x128x16\.F32\b", f16[0]) and not re.search(r"HGMMA\.\w+x8\b|TF32", f16[0])
    assert re.search(r"HGMMA\.64x128x8\.F32\.TF32", tf32[0]) and not re.search(r"HGMMA\.\w+x16", tf32[0])
    for body in (f16[0], tf32[0]):
        assert "UTMALDG" in body and not re.search(r"(?<![A-Z])HMMA", body)


def test_gemm_tc_kernels_do_not_spill(gemm_tc_build):
    ptxas, _ = gemm_tc_build
    blocks = re.split(r"ptxas info\s*: Compiling entry function ", ptxas)[1:]
    seen = 0
    for block in blocks:
        name = block.split("'")[1]
        if not re.search(r"gemm_tc_kernel|split_rows_f16|transpose_split_f16", name):
            continue
        seen += 1
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", block)
        assert m and m.group(1) == "0" and m.group(2) == "0", (name, block)
    assert seen == 4, seen
