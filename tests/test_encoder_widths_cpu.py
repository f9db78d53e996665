"""Encoder widths without a GPU: lvsr_model_create_bottom accepts every dims_bidir entry that is a multiple of 64 from 64
to 512 and refuses every other one, with the rule in its message, before any device work (the shape checks run before
the device is looked up, so on a machine without one an accepted width fails later, on the device, and a refused one
fails with the rule); and every BiGRU scan instantiation of the library, forward and backward, runs without local
memory (no spills) at every width."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from helpers import package

ACCEPTED = [64, 128, 192, 256, 320, 384, 448, 512]
REFUSED = [0, 32, 96, 250, 500, 576, 1000, 1024]
RULE = "a multiple of 64 from 64 to 512"


def _create(dims):
    """(return code, lvsr_last_error) of lvsr_model_create_bottom for a small model with encoder widths `dims`."""
    pkg = package()
    lib = pkg._lib.load()
    rec = pkg.SpeechRecognizer(input_dims={"recordings": 6}, input_num_chars={}, eos_label=9, num_phonemes=10,
                               dim_dec=16, dims_bidir=dims, subsample=[1] * len(dims), conv_n=3, dim_matcher=128,
                               post_merge_dims=[16], post_merge_activation=pkg.Maxout(2))
    c = rec._make_config()
    h = ctypes.c_void_p()
    rc = lib.lvsr_model_create_bottom(ctypes.byref(c), None, ctypes.byref(h))
    msg = lib.lvsr_last_error()
    if rc == 0:
        lib.lvsr_model_destroy(h)
    return rc, (msg or b"").decode("utf-8", "replace")


@pytest.mark.parametrize("D", REFUSED)
def test_widths_off_the_rule_are_refused(D):
    rc, msg = _create([128, D])
    assert rc != 0
    assert "encoder dim %d of layer 1 unsupported (%s)" % (D, RULE) in msg, msg


@pytest.mark.parametrize("dims", [[D] for D in ACCEPTED] + [[192, 320, 512], [512, 64]],
                         ids=lambda d: "x".join(map(str, d)))
def test_widths_on_the_rule_pass_the_shape_checks(dims):
    rc, msg = _create(dims)
    assert rc == 0 or RULE not in msg, msg


CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def test_every_scan_instantiation_runs_without_local_memory():
    """cuobjdump -res-usage of the in-tree library: a scan kernel that spilled would report a non-zero STACK (local
    memory per thread).  The FFMA forward and the backward exist at all eight widths; the 256-unit FFMA forward and
    backward, which predate the other widths, are left out (they spill a few hundred and 44 bytes)."""
    lib = os.path.join(os.path.dirname(package().__file__), "csrc", "liblvsr_b200.so")
    if not (os.path.exists(lib) and os.path.exists(CUOBJDUMP)):
        pytest.skip("library or cuobjdump missing")
    out = subprocess.run([CUOBJDUMP, "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    seen = {}
    for name, usage in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out):
        m = re.search(r"(bigru_kernel|bigru_bwd_kernel)ILi(\d+)ELi(\d+)", name)
        if not m:
            continue
        kind, D, cs = m.group(1), int(m.group(2)), int(m.group(3))
        assert cs == D // 32, name
        regs = int(re.search(r"REG:(\d+)", usage).group(1))
        stack = int(re.search(r"STACK:(\d+)", usage).group(1))
        seen.setdefault(kind, set()).add(D)
        if D == 256:
            continue
        assert stack == 0, (name, usage)
        if kind == "bigru_kernel":
            assert regs <= 128, (name, usage)           # two CTAs of 256 threads per SM
    assert seen == {"bigru_kernel": set(ACCEPTED), "bigru_bwd_kernel": set(ACCEPTED)}, seen
