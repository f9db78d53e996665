"""The unidirectional encoder (net.bidir: False) without a GPU: the float64 oracle of tests/unidirectional_oracle.py
against the bidirectional one, its torch mirror and finite differences, its parameter table against a hand-written
Blocks list; the recognizer's and the C ABI's handling of the flag; the compat plumbing; and the scan instantiations
the flag adds."""
import ctypes
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

import unidirectional_oracle as U
from compat_helpers import COMPAT, write_experiment
from helpers import O, make_recognizer, package

SMALL = dict(num_features=6, dims_bidir=[6], subsample=[1], dim_dec=4, dim_matcher=4, conv_n=2, conv_num_filters=2,
             num_phonemes=5, post_merge_dims=[4], maxout_pieces=2)


def test_one_layer_is_the_forward_half_of_bidirectional():
    cfg = U.make_config(**dict(SMALL, dims_bidir=[8], subsample=[2]))
    bcfg = O.make_config(**dict(SMALL, dims_bidir=[8], subsample=[2]))
    up = U.init_params(cfg, seed=3, scale=10.0)
    bp = O.init_params(bcfg, seed=4, scale=10.0)
    for name, v in up.items():
        if "/with_fork0/" in name:
            bp[name.replace("/with_fork0/", "/bidir0/forward/")] = v
    x, m, _, _ = O.synthetic_batch(bcfg, B=3, T=11, seed=5)
    got, gmask = U.encoder(cfg, up, x, m)
    want, wmask = O.encoder(bcfg, bp, x, m)
    assert got.shape == (6, 3, 8) and want.shape == (6, 3, 16)
    assert np.abs(got - want[:, :, :8]).max() <= 1e-12
    assert np.array_equal(gmask, wmask)


@pytest.mark.parametrize("attention", ["content_and_conv", "content"])
def test_torch_mirror_equals_numpy(attention):
    torch = pytest.importorskip("torch")
    cfg = U.make_config(attention_type=attention, **dict(SMALL, dims_bidir=[6, 4], subsample=[1, 2]))
    params = U.init_params(cfg, seed=1, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=9, seed=2)
    want = U.recognizer_cost(cfg, params, x, m, labels, lm)
    _, _, got = U.cost_and_grads(cfg, params, x, m, labels, lm, return_costs=True)
    assert np.abs(got - want).max() <= 1e-11 * max(1.0, np.abs(want).max())
    att, amask = U.encoder(cfg, params, x, m)
    p = {k: torch.as_tensor(v) for k, v in params.items()}
    tatt, tmask = U._encoder_torch(cfg, p, torch.as_tensor(x), torch.as_tensor(m))
    assert np.abs(tatt.numpy() - att).max() <= 1e-12 and np.array_equal(tmask.numpy(), amask)


def test_autograd_agrees_with_finite_differences():
    pytest.importorskip("torch")
    cfg = U.make_config(**dict(SMALL, dims_bidir=[4, 6], subsample=[1, 2]))
    params = U.init_params(cfg, seed=7, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=2, T=7, seed=8)
    _, grads = U.cost_and_grads(cfg, params, x, m, labels, lm)
    rng = np.random.RandomState(0)
    h = 1e-6
    checked = 0
    for name in params:
        if not name.startswith(U.ENC + "/"):
            continue
        for _ in range(2):
            idx = tuple(rng.randint(s) for s in params[name].shape)
            plus = {k: v.copy() for k, v in params.items()}
            minus = {k: v.copy() for k, v in params.items()}
            plus[name][idx] += h
            minus[name][idx] -= h
            fd = (O.batch_cost(U.recognizer_cost(cfg, plus, x, m, labels, lm)) -
                  O.batch_cost(U.recognizer_cost(cfg, minus, x, m, labels, lm))) / (2 * h)
            assert abs(fd - grads[name][idx]) <= 1e-6 * max(1.0, abs(fd)), (name, idx, fd, grads[name][idx])
            checked += 1
    assert checked == 2 * 7 * 2


def _blocks_table():
    """The Blocks parameter list of a 2-layer [64, 192] forward-only encoder on 40 features, decoder at E = 192."""
    out = []
    for l, (din, D) in enumerate(((40, 64), (64, 192))):
        b = "/recognizer/encoder/with_fork%d" % l
        out += [(b + "/gatedrecurrent.state_to_state", (D, D)), (b + "/gatedrecurrent.state_to_gates", (D, 2 * D)),
                (b + "/gatedrecurrent.initial_state", (D,)), (b + "/fork/fork_inputs.b", (D,)),
                (b + "/fork/fork_inputs.W", (din, D)), (b + "/fork/fork_gate_inputs.b", (2 * D,)),
                (b + "/fork/fork_gate_inputs.W", (din, 2 * D))]
    return out


ARCH = dict(num_features=40, dims_bidir=[64, 192], subsample=[1, 2], dim_dec=128, dim_matcher=128, conv_n=4,
            conv_num_filters=4, num_phonemes=10, post_merge_dims=[128], maxout_pieces=2)


def test_parameter_table_is_the_blocks_list():
    cfg = U.make_config(**ARCH)
    table = list(U.param_shapes(cfg).items())
    enc = [kv for kv in table if kv[0].startswith("/recognizer/encoder/")]
    assert enc == _blocks_table()
    assert table[len(enc):] == [kv for kv in O.param_shapes(O.make_config(**dict(ARCH, dims_bidir=[96], subsample=[1])))
                                .items() if not kv[0].startswith("/recognizer/encoder/")]
    assert dict(table)["/recognizer/generator/att_trans/conv_att/preprocess.W"] == (192, 128)


def _create(rec, bidir):
    pkg = package()
    lib = pkg._lib.load()
    h = ctypes.c_void_p()
    c = rec._make_config()
    rc = lib.lvsr_model_create_encoder(ctypes.byref(c), None, bidir, ctypes.byref(h))
    msg = (lib.lvsr_last_error() or b"").decode("utf-8", "replace")
    if rc == 0:
        lib.lvsr_model_destroy(h)
    return rc, msg


def test_recognizer_takes_the_flag():
    pkg = package()
    cfg = U.make_config(**ARCH)
    rec = make_recognizer(cfg, bidir=False)
    assert rec.bidir is False and rec.net["bidir"] is False and rec.dim_encoded == 192
    assert make_recognizer(cfg).dim_encoded == 384
    import pickle
    assert pickle.loads(pickle.dumps(rec)).dim_encoded == 192
    with pytest.raises(ValueError, match="bidir must be True .* or False"):
        make_recognizer(cfg, bidir="yes")
    rc, msg = _create(rec, 2)
    assert rc != 0 and "bidir 2 unsupported (1: bidirectional encoder, 0: forward-only encoder)" in msg, msg
    rc, msg = _create(rec, 0)                   # past the checks: fails on the device only where there is none
    assert rc == 0 or "bidir" not in msg, msg
    assert "lvsr_model_create_encoder" in pkg._lib.SIGNATURES
    assert pkg._lib.load().lvsr_version() == 104


def test_initial_values_resolve_with_fork_paths():
    cfg = U.make_config(**ARCH)
    rec = make_recognizer(cfg, bidir=False)
    ig = package().IsotropicGaussian
    rec.set_initialization("/recognizer/encoder/with_fork1", weights_init=ig(3.0))
    vals = rec.initial_values(U.param_shapes(cfg), seed=1)
    assert np.std(vals["/recognizer/encoder/with_fork1/fork/fork_inputs.W"]) > 1.0
    assert np.std(vals["/recognizer/encoder/with_fork0/fork/fork_inputs.W"]) < 1.0
    rec.set_initialization("/recognizer/encoder/bidir0", weights_init=ig(3.0))
    with pytest.raises(ValueError, match="no brick of the model at /recognizer/encoder/bidir0"):
        rec.initial_values(U.param_shapes(cfg), seed=1)


def test_compat_carries_the_flag(tmp_path, monkeypatch):
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as LC
    import lvsr.main as LM
    from lvsr.datasets import Data
    pkg = package()
    monkeypatch.setattr(pkg.SpeechRecognizer, "initialize", lambda self, seed=1: None)
    exp = write_experiment(tmp_path)
    cfg = LC.Configuration(exp["base"], "$LVSR/lvsr/configs/schema.yaml", [("net.bidir", "False")])
    assert cfg["net"]["bidir"] is False
    rec = LM.create_model(cfg, Data(**cfg["data"]))
    assert rec.bidir is False and rec.dim_encoded == 128


CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def test_forward_only_scan_instantiations():
    """Every scan kernel exists with one direction beside its two-direction twin; the one-direction FFMA forward scans
    and backward scans use no local memory and the forward ones at most 128 registers, except at 256 units, whose
    two-direction FFMA kernels already spill (the tensor-core scan runs that width)."""
    lib = package()._lib.LIB_PATH
    if not (os.path.exists(lib) and os.path.exists(CUOBJDUMP)):
        pytest.skip("library or cuobjdump missing")
    out = subprocess.run([CUOBJDUMP, "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    seen = {}
    for name, usage in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out):
        m = re.search(r"(bigru_kernel|bigru_bwd_kernel)ILi(\d+)ELi(\d+)ELi(\d+)E", name)
        mm = re.search(r"bigru_mma_kernelILi(\d+)ELi(\d+)E", name)
        if mm:
            seen.setdefault("mma", set()).add(int(mm.group(2)))
            continue
        if not m:
            continue
        kind, D, ndir = m.group(1), int(m.group(2)), int(m.group(4))
        seen.setdefault((kind, ndir), set()).add(D)
        if ndir != 1 or D == 256:
            continue
        assert int(re.search(r"STACK:(\d+)", usage).group(1)) == 0, (name, usage)
        if kind == "bigru_kernel":
            assert int(re.search(r"REG:(\d+)", usage).group(1)) <= 128, (name, usage)
    widths = {64, 128, 192, 256, 320, 384, 448, 512}
    for kind in ("bigru_kernel", "bigru_bwd_kernel"):
        assert seen[(kind, 1)] == seen[(kind, 2)] == widths, seen
    assert seen["mma"] == {1, 2}, seen
