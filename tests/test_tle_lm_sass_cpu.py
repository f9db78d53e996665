"""Resources of the readout kernel's instantiations in the built library (no GPU needed: cuobjdump -res-usage on the
in-tree .so).  The task-loss readout fused with a language model is an instantiation of its own, so the
log-likelihood readout and the task-loss readout without a language model keep the code they had before it was
added: 40 and 39 registers (sm_90a, CUDA 12.9), and none of the three uses local memory."""
import os
import re
import shutil
import subprocess

import pytest

from helpers import package

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
LL = "14readout_kernelILb0ELb0EEEvNS_11ReadoutArgsE"
TLE = "14readout_kernelILb1ELb0EEEvNS_11ReadoutArgsE"
TLE_LM = "14readout_kernelILb1ELb1EEEvNS_11ReadoutArgsE"


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
    hits = {k: v for k, v in usage.items() if k.endswith(needle)}
    assert len(hits) == 1, (needle, sorted(hits))
    return next(iter(hits.values()))


def test_readout_has_three_instantiations(usage):
    assert len([k for k in usage if "14readout_kernelI" in k]) == 3


@pytest.mark.parametrize("kernel", [LL, TLE, TLE_LM])
def test_no_local_memory(usage, kernel):
    u = _find(usage, kernel)
    assert u["LOCAL"] == 0 and u["STACK"] == 0, (kernel, u)


@pytest.mark.parametrize("kernel,regs", [(LL, 40), (TLE, 39)])
def test_readouts_without_the_fused_task_loss_keep_their_registers(usage, kernel, regs):
    assert _find(usage, kernel)["REG"] == regs
