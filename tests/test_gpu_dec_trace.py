"""The persistent decoder's debug trace (LVSR_DEC_TRACE) and the switch to the step-wise kernels (LVSR_NO_DEC_SCAN).

The trace buffer is taken from the workspace behind the decoder's hand-over buffers, and the kernel stamps it beside
its hand-overs.  A traced call must therefore compute what an untraced one computes, bit for bit, on the same plan,
and print its phase times on stderr.  Both layouts the planner can choose are run, islands (B >= 16) and global
(B < 16), with the LVSR_DEC_CHECK post-condition on.  One BiGRU(128) layer without subsampling: T' = T, and the
tests pass `attended` directly.
"""
import math
import re

import numpy as np
import pytest

from helpers import O, f32, make_recognizer

pytestmark = pytest.mark.gpu

ARCH = dict(num_features=40, dims_bidir=[128], subsample=[1], dim_dec=128, dim_matcher=256, conv_n=8,
            conv_num_filters=10, num_phonemes=32, post_merge_dims=[128], maxout_pieces=2)
SWITCHES = ("LVSR_DEC_CS", "LVSR_DEC_LAYOUT", "LVSR_DEC_HANDLER", "LVSR_ATT_CS", "LVSR_NO_DEC_SCAN", "LVSR_DEC_TRACE",
            "LVSR_DEC_CHECK")
PHASES = {"CTA first": ("A", "syncA", "B1", "sync1", "B2", "sync2", "B3", "sync3"),
          "CTA last": ("A", "syncA", "B1", "sync1", "B2", "sync2", "B3", "sync3"),
          "attention row 0": ("stage", "conv", "energy", "stats", "ctx", "exchange", "combine"),
          "gate tile": ("wait_x", "products", "sums", "epilogue")}


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


@pytest.fixture
def env(monkeypatch):
    """No plan-forcing switch from the caller's environment; the post-condition on."""
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("LVSR_DEC_CHECK", "1")
    return monkeypatch


def _case(B, Tp, L, seed):
    """A recognizer and device inputs: attended [T',B,E] in (-1, 1), ragged lengths (one row full), labels and a label
    mask with trailing zeros."""
    torch = _torch()
    cfg = O.make_config(**ARCH)
    rec = make_recognizer(cfg, {k: f32(v) for k, v in O.init_params(cfg, seed=seed, scale=10.0).items()})
    rng = np.random.RandomState(seed)
    lens = rng.randint(int(math.ceil(0.6 * Tp)), Tp + 1, size=B)
    lens[rng.randint(B)] = Tp
    att = torch.as_tensor(rng.uniform(-1, 1, size=(Tp, B, O.dim_encoded(cfg))), dtype=torch.float32, device="cuda")
    attm = torch.as_tensor(np.arange(Tp)[:, None] < lens[None, :], dtype=torch.float32, device="cuda")
    labels = rng.randint(0, ARCH["num_phonemes"] - 1, size=(L, B)).astype(np.int64)
    lm = (np.arange(L)[:, None] < rng.randint(L - 3, L + 1, size=B)[None, :]).astype(np.float64)
    return rec, (labels, lm, att, attm)


def _run(rec, inputs):
    out = rec.cost_matrix(*inputs, return_all=True)
    return {k: v.cpu().numpy() for k, v in out.items()}, rec.decoder_plan(), rec.launch_status()


@pytest.mark.parametrize("layout,B", [("islands", 16), ("global", 6)])
def test_trace_leaves_every_output_and_the_plan_unchanged(env, capfd, layout, B):
    rec, inputs = _case(B, Tp=40, L=12, seed=B)
    env.setenv("LVSR_DEC_LAYOUT", layout)
    want, want_plan, status = _run(rec, inputs)
    assert status == (0, 0)
    assert want_plan["ran"] and want_plan["kernel"] == "dec_scan", want_plan
    assert (want_plan["nisl"] > 0) == (layout == "islands"), want_plan
    capfd.readouterr()
    env.setenv("LVSR_DEC_TRACE", "1")
    got, plan, status = _run(rec, inputs)
    err = capfd.readouterr().err
    assert status == (0, 0)
    assert plan == want_plan
    for k in want:
        assert np.array_equal(got[k].view(np.uint32), want[k].view(np.uint32)), k

    lines = [ln for ln in err.splitlines() if ln.startswith("[dec_scan trace] ")]
    heads = [ln[len("[dec_scan trace] "):].partition(":")[0] for ln in lines]
    assert sorted(heads) == sorted(list(PHASES) + ["end of attention vs row 0 (us)"]), err
    for ln in lines:
        head, _, body = ln[len("[dec_scan trace] "):].partition(":")
        if head == "end of attention vs row 0 (us)":
            ends = [float(x) for x in body.split()]
            assert len(ends) == B and all(math.isfinite(x) for x in ends), ln
            continue
        times = re.findall(r"(\w+)=([^ ]+)us", body)
        assert tuple(name for name, _ in times) == PHASES[head], ln
        assert all(math.isfinite(float(t)) and float(t) >= 0 for _, t in times), ln


def test_stepwise_call_after_the_persistent_decoder_reports_a_clean_step_wise_plan(env):
    """The status word is zeroed and the plan report reset on every call, also when the call does not plan."""
    rec, inputs = _case(16, Tp=40, L=12, seed=3)
    _, plan, status = _run(rec, inputs)
    assert plan["ran"] and status == (0, 0), plan
    env.setenv("LVSR_NO_DEC_SCAN", "1")
    _, plan, status = _run(rec, inputs)
    assert status == (0, 0)
    assert plan["ran"] is False and plan["kernel"] == "stepwise", plan
    assert plan["att_cs"] > 0, plan
    assert all(v == 0 for k, v in plan.items() if k not in ("ran", "kernel", "att_cs")), plan
