"""The built library really contains the Hopper code paths the design names (no GPU needed: cuobjdump on the in-tree .so).
SASS mnemonics: wgmma.mma_async -> HGMMA, TMA -> UTMALDG, mma.sync -> HMMA."""
import os
import re
import shutil
import subprocess

import pytest

from helpers import package

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.fixture(scope="module")
def sass():
    lib = package()._lib.LIB_PATH
    if not os.path.exists(lib) or not os.path.exists(CUOBJDUMP):
        pytest.skip("library or cuobjdump missing")
    out = subprocess.run([CUOBJDUMP, "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name and "/*" in line:
            funcs[name].append(line)
    return funcs


def _body(funcs, needle):
    hits = [k for k in funcs if needle in k]
    assert hits, "no kernel named *%s* in the library" % needle
    return {k: "\n".join(funcs[k]) for k in hits}


def test_library_is_sm90a_only():
    lib = package()._lib.LIB_PATH
    if not os.path.exists(lib) or not os.path.exists(CUOBJDUMP):
        pytest.skip("library or cuobjdump missing")
    out = subprocess.run([CUOBJDUMP, "-lelf", lib], capture_output=True, text=True, check=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_fork_gemm_runs_on_wgmma_with_tma(sass):
    for name, body in _body(sass, "gemm_tc_kernel").items():
        assert re.search(r"HGMMA\.64x(128|256)x", body), name  # wgmma.mma_async, one m64 slab per consumer warpgroup
        assert "UTMALDG" in body, name                       # cp.async.bulk.tensor
        assert not re.search(r"(?<![A-Z])HMMA", body), name   # not the legacy tensor path


def test_bigru_recurrence_runs_on_tensor_cores_with_register_reallocation(sass):
    for name, body in _body(sass, "bigru_mma_kernel").items():
        assert body.count("HMMA.16816.F32") >= 48, name      # 3 products x 8 k-steps x 2 MMAs per warp
        assert "USETMAXREG" in body, name                     # setmaxnreg: registers move to the MMA warps
        assert "STAS" in body, name                           # st.async into the peers' shared memory
        assert "BAR.ARV" in body, name                        # MMA warps arrive, never wait for the elementwise warps
        assert not re.search(r"\bLDL\b|\bSTL\b", body), name  # 192 weight registers per lane without a spill


def test_persistent_decoder_uses_cluster_exchange_and_tensor_cores(sass):
    for name, body in _body(sass, "dec_scan_kernel").items():
        assert "HMMA" in body, name                           # handler product of the location features
        assert "UCGABAR" in body or "CGABAR" in body, name    # cluster barrier of a row's CTAs
