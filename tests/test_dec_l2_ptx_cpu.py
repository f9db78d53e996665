"""The persistent decoder can load P and H with an L2 cache policy, and nothing else about the kernels changes (no GPU
needed: dec_scan.cu and attention.cu compiled on their own for sm_90a).

In the instantiations with HINT = true, the energy loop's P loads and the context loop's H loads of dec_scan_kernel
and dec_content_kernel are ld.global.nc.L1::no_allocate.L2::cache_hint with the policy made once at kernel entry
(createpolicy.fractional); with HINT = false, and in the step-wise att_step_kernel, they are plain loads.  The policy
lives in the load's uniform descriptor, so every instantiation stays at the 128-register cap with no more spill traffic
than before: 4 and 12 bytes of spill stores with the compact and the padded handler copy, none for content attention."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "attention-lvcsr_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
         "-I" + os.path.join(CSRC, "..", "..", "include"), "-I" + CSRC]


def _ptx_functions(ptx):
    """{entry name: body} of a PTX module"""
    out = {}
    for m in re.finditer(r"\.entry\s+(\S+?)\s*\(", ptx):
        start = m.end()
        nxt = re.search(r"\.entry\s", ptx[start:])
        out[m.group(1)] = ptx[start:start + nxt.start()] if nxt else ptx[start:]
    return out


@pytest.fixture(scope="module")
def compiled():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc missing")
    with tempfile.TemporaryDirectory() as tmp:
        res = {}
        for src in ("dec_scan", "attention"):
            ptx = os.path.join(tmp, src + ".ptx")
            subprocess.run([NVCC, *FLAGS, "-ptx", os.path.join(CSRC, src + ".cu"), "-o", ptx], check=True)
            with open(ptx) as f:
                res[src] = _ptx_functions(f.read())
        ptxas = subprocess.run([NVCC, *FLAGS, "-Xptxas", "-v", "-c", os.path.join(CSRC, "dec_scan.cu"), "-o",
                                os.path.join(tmp, "dec_scan.o")], capture_output=True, text=True, check=True).stderr
    return res, ptxas


def _hinted(body):
    return re.findall(r"ld\.global\.nc\.L1::no_allocate\.L2::cache_hint\.(v2|v4)\.f32", body)


# mangled template arguments of the persistent decoder's kernels: dec_scan_kernel<COMPACT, HINT>, dec_content_kernel<HINT>
HINTED = ("dec_scan_kernelILb0ELb1E", "dec_scan_kernelILb1ELb1E", "dec_content_kernelILb1E")
PLAIN = ("dec_scan_kernelILb0ELb0E", "dec_scan_kernelILb1ELb0E", "dec_content_kernelILb0E")
PLAIN_LOAD = r"ld\.global\.nc\.v[24]\.f32"


def _find(funcs, key):
    names = [k for k in funcs if key in k]
    assert len(names) == 1, (key, sorted(funcs))
    return funcs[names[0]]


def test_decoder_kernels_load_p_and_h_with_the_l2_policy(compiled):
    funcs, _ = compiled
    for key in HINTED:
        body = _find(funcs["dec_scan"], key)
        assert "createpolicy.fractional.L2::evict_normal.L2::evict_first.b64" in body, key
        kinds = _hinted(body)
        assert "v2" in kinds and "v4" in kinds, (key, kinds)    # P tiles (float2) and H rows (float4)
        assert not re.search(PLAIN_LOAD, body), key              # no P or H load is left without the policy
    for key in PLAIN:
        body = _find(funcs["dec_scan"], key)
        assert "cache_hint" not in body and "createpolicy" not in body, key
        assert re.search(PLAIN_LOAD, body), key


def test_stepwise_attention_keeps_plain_loads(compiled):
    funcs, _ = compiled
    names = [k for k in funcs["attention"] if "att_step_kernel" in k]
    assert names, sorted(funcs["attention"])
    for name in names:
        body = funcs["attention"][name]
        assert "cache_hint" not in body and "createpolicy" not in body, name
        assert re.search(PLAIN_LOAD, body), name


def test_decoder_kernels_keep_their_registers_and_spills(compiled):
    _, ptxas = compiled
    seen = {}
    for block in re.split(r"ptxas info\s*: Compiling entry function ", ptxas)[1:]:
        name = block.split("'")[1]
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", block)
        r = re.search(r"Used (\d+) registers", block)
        for key in HINTED + PLAIN:
            if key in name:
                seen[key] = (int(r.group(1)), int(m.group(1)), int(m.group(2)))
    assert len(seen) == 6, seen
    # spill stores: 4 bytes for the compact handler copy, 12 for the padded one, none for content attention
    limits = {"dec_scan_kernelILb1E": 4, "dec_scan_kernelILb0E": 12, "dec_content_kernel": 0}
    for key, (regs, stores, _) in seen.items():
        assert regs == 128, (key, seen)
        assert stores <= next(v for k, v in limits.items() if key.startswith(k)), (key, seen)
