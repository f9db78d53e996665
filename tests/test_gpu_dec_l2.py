"""The persistent decoder's L2 priority of P and H (dec_scan.cu l2_plan, LVSR_DEC_L2) changes which lines the L2 keeps,
never what is computed: every output is bit-identical with the hints off, at the default and at forced fractions, and
so are a training step's gradients.  decoder_plan()["l2_evict_first_kb"] reports the KB of P and H per step loaded
evict-first: by default all of both when together they exceed the L2 (counted over the positions a step reads), 0 when
they fit and under the window-around priors; under LVSR_DEC_L2=<fP>,<fH> the shares 1 - fP of P and 1 - fH of H."""
import numpy as np
import pytest

import bench
from helpers import O, make_recognizer, package

pytestmark = pytest.mark.gpu


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _expected_kb(torch, Tp, B, M, E, fp=0.0, fh=0.0):
    """the default plan's report (fp = fh = 0), or a forced setting's"""
    bp, bh = float(Tp) * B * M * 4, float(Tp) * B * E * 4
    return int(((1 - fp) * bp + (1 - fh) * bh) / 1024)


def _l2_bytes(torch):
    return torch.cuda.get_device_properties(0).L2_cache_size


def _model(prior=None):
    cfg = O.make_config(**bench.NET)
    if prior is not None:
        cfg["prior"] = prior
    rec = make_recognizer(cfg)
    rec.set_parameter_values(bench.init_values(rec.parameter_shapes()))
    return rec


def _cost_matrix(rec, B, T, L, seed=1234):
    x, m, labels, lm = bench.synthetic_batch(B, T, 40, L, 32, seed=seed)
    att, attm = rec.encode(x, m)
    return att, lambda: rec.cost_matrix(labels, lm, att, attm, return_all=True)


def test_outputs_are_bit_identical_under_every_setting_at_the_metric_shape(monkeypatch):
    torch = _torch()
    monkeypatch.setenv("LVSR_DEC_CHECK", "1")
    W = bench.WORKLOAD
    rec = _model()
    att, call = _cost_matrix(rec, W["B"], W["T"], W["L"])
    Tp, B, E = att.shape
    M = bench.NET["dim_matcher"]
    runs = {}
    for setting in ("off", None, "1,0", "0.5,0.3"):
        if setting is None:
            monkeypatch.delenv("LVSR_DEC_L2", raising=False)
        else:
            monkeypatch.setenv("LVSR_DEC_L2", setting)
        runs[setting] = {k: v.clone() for k, v in call().items()}
        plan = rec.decoder_plan()
        assert plan["ran"] and plan["kernel"] == "dec_scan" and rec.launch_status() == (0, 0), plan
        runs[setting]["kb"] = plan["l2_evict_first_kb"]
    assert runs["off"]["kb"] == 0
    assert (Tp * B * (M + E) * 4 > _l2_bytes(torch)) and runs[None]["kb"] == _expected_kb(torch, Tp, B, M, E)
    assert runs["1,0"]["kb"] == _expected_kb(torch, Tp, B, M, E, 1, 0) == int(Tp * B * E * 4 / 1024)
    assert runs["0.5,0.3"]["kb"] == _expected_kb(torch, Tp, B, M, E, 0.5, 0.3)
    for setting in (None, "1,0", "0.5,0.3"):
        for k in ("costs", "weights", "energies", "states", "weighted_averages"):
            assert torch.equal(runs[setting][k], runs["off"][k]), (setting, k)


def test_hints_are_off_where_plain_lru_keeps_the_lines(monkeypatch):
    torch = _torch()
    monkeypatch.setenv("LVSR_DEC_CHECK", "1")
    monkeypatch.delenv("LVSR_DEC_L2", raising=False)
    # config 2 (B=32 x T=800): P and H together fit in the L2
    rec = _model()
    att, call = _cost_matrix(rec, 32, 800, 100)
    call()
    plan = rec.decoder_plan()
    assert plan["ran"] and plan["l2_evict_first_kb"] == 0, plan
    assert att.shape[0] * 32 * (bench.NET["dim_matcher"] + att.shape[2]) * 4 <= _l2_bytes(torch)
    # the window-around priors: each step's window follows the alignment
    rec = _model(dict(type="window_around_median", before=100, after=100))
    _, call = _cost_matrix(rec, 64, 1000, 125)
    call()
    plan = rec.decoder_plan()
    assert plan["ran"] and plan["l2_evict_first_kb"] == 0, plan


def test_invalid_setting_is_an_error(monkeypatch):
    _torch()
    rec = _model()
    _, call = _cost_matrix(rec, 16, 64, 8)
    for bad in ("on", "1", "1.5,0", "0.5,0.1,0.2", "-0.1,0"):
        monkeypatch.setenv("LVSR_DEC_L2", bad)
        with pytest.raises(RuntimeError, match="LVSR_DEC_L2"):
            call()


def test_training_step_gradients_are_bit_identical_with_the_plan_on_and_off(monkeypatch):
    torch = _torch()
    monkeypatch.setenv("LVSR_DEC_CHECK", "1")
    W = bench.TRAIN_WORKLOAD
    rec = _model()
    lib = package()._lib.load()
    dev = torch.device("cuda", 0)
    x, m, labels, lm = bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"], seed=4321)
    xd, md, yd, ymd = (torch.as_tensor(a, device=dev) for a in (x, m, labels, lm))
    h = rec._require_ready()
    out = {}
    for setting in ("off", None):
        if setting is None:
            monkeypatch.delenv("LVSR_DEC_L2", raising=False)
        else:
            monkeypatch.setenv("LVSR_DEC_L2", setting)
        g = torch.zeros(int(lib.lvsr_model_flat_size(h)), device=dev)
        c = torch.zeros(1, device=dev)
        rc = lib.lvsr_train_cost_and_grads(h, xd.data_ptr(), md.data_ptr(), yd.data_ptr(), ymd.data_ptr(), W["T"],
                                           W["B"], W["L"], 1.0 / W["B"], c.data_ptr(), g.data_ptr(), rec._stream())
        assert rc == 0, lib.lvsr_last_error()
        torch.cuda.synchronize(dev)
        out[setting] = (c, g, rec.decoder_plan()["l2_evict_first_kb"])
    assert out["off"][2] == 0
    # configs[3]: T' = 375, P and H 49 MB each
    Tp = rec.encoded_length(W["T"])
    assert out[None][2] == _expected_kb(torch, Tp, W["B"], bench.NET["dim_matcher"], 2 * bench.NET["dims_bidir"][-1]) > 0
    assert torch.equal(out[None][0], out["off"][0])
    assert torch.equal(out[None][1], out["off"][1])
    assert np.isfinite(out["off"][0].item())
