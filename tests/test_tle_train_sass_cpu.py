"""Resources of the task-loss training kernels in the built library (no GPU needed: cuobjdump -res-usage on the
in-tree .so): the loss gradient, the greedy pick and both instantiations of the readout backward run without local
memory, and making the readout backward a template on the emitter left the log-likelihood instantiation at the 40
registers of the kernel it replaced (sm_90a, CUDA 12.9)."""
import os
import re
import shutil
import subprocess

import pytest

from helpers import package

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
LL_READOUT_BWD = "_ZN4lvsr5train18readout_bwd_kernelILb0EEEvNS0_14ReadoutBwdArgsE"
TLE_READOUT_BWD = "_ZN4lvsr5train18readout_bwd_kernelILb1EEEvNS0_14ReadoutBwdArgsE"


@pytest.fixture(scope="module")
def usage():
    lib = package()._lib.LIB_PATH
    if not os.path.exists(lib) or not os.path.exists(CUOBJDUMP):
        pytest.skip("library or cuobjdump missing")
    out = subprocess.run([CUOBJDUMP, "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
        elif name and "REG:" in line:
            funcs[name] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
            name = None
    return funcs


def _find(usage, needle):
    hits = {k: v for k, v in usage.items() if needle in k}
    assert len(hits) == 1, (needle, sorted(hits))
    return next(iter(hits.values()))


@pytest.mark.parametrize("kernel", ["tle_grad_kernel", "tle_greedy_pick_kernel", LL_READOUT_BWD, TLE_READOUT_BWD])
def test_no_local_memory(usage, kernel):
    u = _find(usage, kernel)
    assert u["LOCAL"] == 0 and u["STACK"] == 0, (kernel, u)


def test_log_likelihood_readout_backward_keeps_its_registers(usage):
    assert _find(usage, LL_READOUT_BWD)["REG"] == 40
