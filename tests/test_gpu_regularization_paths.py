"""Dropout, weight noise and the alignment penalty on the kernels the training step takes beyond the small encoder of
test_gpu_regularization.py: the tensor-core BiGRU scan and its backward (D = 256) with tensor-core weight gradients
(T*B >= 2048 rows) and again with them off (LVSR_NO_TC_GEMM=1), the FFMA scan at widths 192 and 448, a bottom MLP of
64-multiple widths, the encoder projection streamed beside the previous scan, the persistent decoder and the
step-wise one, content attention and the logistic and relu normalisers at R = L*B > 1024 decoder rows, and the
longest T' the attention backward takes.  Each case asserts the plan it is for, so a fallback fails.

The draws the float64 oracle (tests/regularization_oracle.py) is given are tests/draws_oracle.py's, derived from
Philox and Box-Muller, not the library's replay: a case passes only if the training step drew them with the seed,
update 0 and utterance offset 0 it was given, on every element.

Weight noise and dropout are compared by cost and every gradient at test_gpu_regularization.py's bar.  The penalty
is compared by its sum P, which is continuous, to a bar derived from the float32 cumsum error (_penalty_bar); a
penalty case with another regulariser also compares that regulariser's gradients with penalty_coof = 0.

The penalty's gradient is not compared at these shapes, because no point was found where it is tie-free.  It depends
on every comparison c_i[t] >= c_{i-1}[t], and float32 alignments may take either side of one within about 2e-5.
With initial weights the alignments are diffuse, and thousands of live comparisons fall within 1e-7 of a tie
(_margin prints the closest).  Multiplying the attention's energy vector by 100 or 300 makes them peaked, and then
every comparison with c (1 - c) > 1e-3 clears 1e-4 for conv and content attention (not for the logistic
normaliser: margins 1e-10 to 4e-7 over four seeds).  But tens of thousands of comparisons with c (1 - c) <= 1e-3
remain within 1e-4 of a tie.  Taking those the other way moves the float64 gradient by 6e-4 of its largest entry
(B = 32, T' = 48), six times the bar, and moving only those within 1e-6 still moves it by 3e-5.  A gradient
comparison there would test float32's tie decisions, not the kernels.  The penalty gradient is compared at
test_gpu_regularization.py's small shapes."""
from collections import OrderedDict

import numpy as np
import pytest

import bottom_oracle as BO
import content_oracle as CO
import draws_oracle as D
import regularization_oracle as RO
from helpers import O, bottom_params, bottom_recognizer, check_overlap_claims, f32, make_recognizer, package

pytestmark = pytest.mark.gpu

BASE = dict(num_features=40, dims_bidir=[256], subsample=[1], dim_dec=128, dim_matcher=256, conv_n=8,
            conv_num_filters=10, num_phonemes=32, post_merge_dims=[128], maxout_pieces=2)
LEVEL, COOF, SEED = 0.05, 0.5, 9
TOL, ATOL_FRAC = 1e-4, 1e-6
# W_REL: the relative error of the float32 alignments (2e-5, measured at encoded widths 128 to 1024).  OMEGA: the
# c (1 - c) above which _margin counts a comparison.
W_REL = 2e-5
OMEGA = 1e-3


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _params(cfg, seed):
    if cfg.get("bottom"):
        return bottom_params(cfg, seed)
    init = CO.init_params if cfg.get("attention_type") == "content" else O.init_params
    return OrderedDict((k, f32(v)) for k, v in init(cfg, seed=seed, scale=10.0).items())


def _algorithm(cfg, params, reg):
    pkg = package()
    rec = bottom_recognizer(cfg, params) if cfg.get("bottom") else make_recognizer(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]),
                               regularization=dict(reg, seed=SEED))
    algo.initialize()
    return algo, rec


def _oracle_draws(algo, rec, cfg, reg, batch):
    """(multiplier [T, B, F], {name: eps}) of update 0 from draws_oracle (None where the regulariser is off)."""
    x = batch[0]
    mult = eps = None
    if reg.get("dropout"):
        F = cfg["bottom"]["dims"][-1] if cfg.get("bottom") else cfg["num_features"]
        mult = D.dropout_multiplier(SEED, 0, 0, x.shape[0], x.shape[1], F).astype(np.float64)
    if reg.get("noise"):
        off = algo._offsets()
        names, spans = list(off), list(off.values())
        flat, _ = D.weight_noise_eps(SEED, 0, spans, algo._n, [RO.is_noise_subject(k) for k in names])
        shapes = rec.parameter_shapes()
        eps = OrderedDict((k, flat[o:o + c].reshape(shapes[k])) for k, (o, c) in off.items())
    return mult, eps


def _margin(w, labels_mask):
    """(smallest |c_i[t] - c_{i-1}[t]|, number of comparisons) over the live comparisons where a flip of the
    indicator would matter: max(c_i (1 - c_i), c_{i-1} (1 - c_{i-1})) > OMEGA."""
    c = np.cumsum(w, axis=2)
    h = np.maximum(c[1:] * (1 - c[1:]), c[:-1] * (1 - c[:-1]))
    live = (h > OMEGA) & (np.asarray(labels_mask)[1:, :, None] > 0)
    d = np.abs(c[1:] - c[:-1])[live]
    return (float(d.min()) if d.size else np.inf), int(d.size)


def _penalty_bar(w, labels_mask):
    """Absolute bound on |P(float32) - P(float64)|: each live term max(c_i - c_{i-1}, 0) moves by at most
    |dc_i| + |dc_{i-1}|, and a float32 cumsum of weights with relative error W_REL over T' positions is off by at most
    (W_REL + T' 2^-24) c."""
    c = np.cumsum(w, axis=2)
    live = np.asarray(labels_mask, np.float64)[1:, :, None]
    return (W_REL + w.shape[2] * 2.0 ** -24) * float(((c[1:] + c[:-1]) * live).sum())


def _check_gradients(grads, want):
    gmax = max(np.abs(v).max() for v in want.values())
    worst, bad = 0.0, {}
    for k, v in want.items():
        scale = max(np.abs(v).max(), 1e-30)
        e = float(np.abs(grads[k].astype(np.float64) - v).max() / scale)
        bar = TOL + ATOL_FRAC * gmax / scale
        worst = max(worst, e / bar)
        if e > bar:
            bad[k] = e
    assert not bad, bad
    return worst


def _run(cfg, reg, B, T, seed, L=None):
    """The training step's cost and gradients against the oracle on draws_oracle's draws; returns the recognizer of
    the last run (for plan assertions) and the batch.

    With the penalty: its sum P against the oracle's to _penalty_bar, and the step runs a second time with
    penalty_coof = 0, where the gradients of the other regulariser (if any) are compared."""
    params = _params(cfg, seed)
    kw = dict(label_div=int(np.ceil(T / (L - 1)))) if L else {}
    batch = O.synthetic_batch(cfg, B=B, T=T, seed=seed + 1, **kw)
    if L:
        assert batch[2].shape[0] == L
    if cfg.get("bottom"):
        assert not BO.kinks(cfg, params, batch[0], batch[1])
    p64 = OrderedDict((k, v.astype(np.float64)) for k, v in params.items())
    coof = reg.get("penalty_coof", 0.0)
    algo, rec = _algorithm(cfg, params, reg)
    cost, grads = algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
    mult, eps = _oracle_draws(algo, rec, cfg, reg, batch)
    want_cost, want, pen, w = RO.cost_and_grads(cfg, p64, *batch, mult=mult, eps=eps, level=LEVEL, coof=coof,
                                                return_penalty=True)
    assert abs(cost - want_cost) <= 1e-4 * abs(want_cost), (cost, want_cost)
    if coof:
        got_pen = float(algo._buf[algo._n + 2].item())
        margin, n = _margin(w, batch[3])
        bar = _penalty_bar(w, batch[3])
        print("penalty %.6f (float64 %.6f, bar %.1e), R = %d rows; tie margin %.1e over %d comparisons"
              % (got_pen, pen, bar, batch[2].size, margin, n))
        assert pen > 0 and abs(got_pen - pen) <= bar, (got_pen, pen, bar)
        rest = {k: v for k, v in reg.items() if k != "penalty_coof"}
        if not rest:
            return rec, batch
        algo, rec = _algorithm(cfg, params, rest)
        cost, grads = algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
        want_cost, want = RO.cost_and_grads(cfg, p64, *batch, mult=mult, eps=eps, level=LEVEL)
        assert abs(cost - want_cost) <= 1e-4 * abs(want_cost), (cost, want_cost)
    worst = _check_gradients(grads, want)
    print("cost %.6f (float64 %.6f); worst gradient error / bar %.2f" % (cost, want_cost, worst))
    # the regulariser acted: the clean oracle differs
    _, clean = RO.cost_and_grads(cfg, p64, *batch)
    assert any(np.abs(clean[k] - grads[k]).max() > 1e-2 * np.abs(clean[k]).max() for k in clean)
    return rec, batch


# ---- the encoder's kernels ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("tc", [True, False], ids=["tc_gemm", "no_tc_gemm"])
@pytest.mark.parametrize("reg", [dict(noise=LEVEL), dict(dropout=True)], ids=["noise", "dropout"])
def test_mma_scan_and_weight_gradients_at_2560_rows(reg, tc, monkeypatch):
    """BiGRU(256) at B = 16, T = 160: the tensor-core scan and its backward, and the encoder's weight gradients over
    2560 rows on tensor cores with split K (or on FFMA under LVSR_NO_TC_GEMM=1), on the noisy copy of the
    parameters or on the dropped-out input."""
    _torch()
    if not tc:
        monkeypatch.setenv("LVSR_NO_TC_GEMM", "1")
    rec, _ = _run(O.make_config(**BASE), reg, B=16, T=160, seed=11)
    p, = rec.encoder_plan()
    assert p["bigru"] == "mma" and p["tape"] and p["T"] == 160, p
    if tc:
        assert p["wgrad"] == "tc" and p["wgrad_splits"] > 1, p
    else:
        assert p["wgrad"] == "ffma", p


@pytest.mark.parametrize("width", [192, 448])
def test_ffma_scan_widths_with_weight_noise(width):
    _torch()
    rec, _ = _run(O.make_config(**dict(BASE, dims_bidir=[width])), dict(noise=LEVEL), B=8, T=80, seed=21)
    p, = rec.encoder_plan()
    assert p["bigru"] == "ffma" and p["tape"], p


def test_bottom_mlp_of_64_multiple_widths_with_dropout():
    """A bottom MLP [256, 128] (tanh, which has no kink for a float32 forward to land on the other side of): the
    dropout multiplier over its 128-wide output, and the backward through the mask into both layers."""
    _torch()
    cfg = BO.make_config(O.make_config(**BASE), [256, 128], "tanh")
    rec, _ = _run(cfg, dict(dropout=True), B=16, T=160, seed=31)
    p = rec.encoder_plan()[0]
    assert p["bigru"] == "mma" and p["dx"] == "tc", p


def test_streamed_encoder_projection_with_weight_noise():
    """Two layers, the second's projection streamed beside the first's scan, both reading the noisy copy."""
    _torch()
    cfg = O.make_config(**dict(BASE, dims_bidir=[256, 256], subsample=[1, 2], dim_matcher=256, conv_n=100,
                               dim_dec=256, post_merge_dims=[256]))
    rec, _ = _run(cfg, dict(noise=LEVEL), B=5, T=40, seed=41)
    plan = rec.encoder_plan()
    assert [(p["overlap"], p["tape"]) for p in plan] == [(False, True), (True, True)], plan
    check_overlap_claims(rec, plan, 5, cfg["subsample"])


# ---- the decoder and the attention with the penalty ---------------------------------------------------------------

def test_penalty_on_the_persistent_decoder_in_islands():
    """B = 32: the persistent decoder's taped forward in 16-row islands: P on the noisy copy of the parameters, and the
    weight-noise gradients without the penalty."""
    _torch()
    rec, _ = _run(O.make_config(**dict(BASE, dims_bidir=[128])), dict(penalty_coof=COOF, noise=LEVEL), B=32, T=48,
                  seed=51)
    plan = rec.decoder_plan()
    print("decoder plan", plan)
    assert plan["ran"] and plan["kernel"].startswith("dec_scan") and plan["nisl"] >= 2, plan
    assert rec.launch_status() == (0, 0)


def test_penalty_on_the_stepwise_decoder(monkeypatch):
    """The step-wise decoder (LVSR_NO_DEC_SCAN=1) takes the taped forward of 72 rows: P with dropout, and the
    dropout gradients without the penalty."""
    _torch()
    monkeypatch.setenv("LVSR_NO_DEC_SCAN", "1")
    rec, _ = _run(O.make_config(**dict(BASE, dims_bidir=[128])), dict(penalty_coof=COOF, dropout=True), B=72, T=48,
                  seed=61)
    plan = rec.decoder_plan()
    assert not plan["ran"] and plan["kernel"] == "stepwise", plan


@pytest.mark.parametrize("kind", ["content", "logistic", "relu"])
def test_penalty_over_more_than_1024_decoder_rows(kind):
    """R = L*B = 16 * 70 = 1120 rows: the forward's penalty sum over more than 1024 rows."""
    _torch()
    base = dict(BASE, dims_bidir=[128])
    cfg = CO.make_config(**base) if kind == "content" else O.make_config(**dict(base, energy_normalizer=kind))
    _, batch = _run(cfg, dict(penalty_coof=COOF), B=16, T=138, seed=71, L=70)
    assert batch[2].size > 1024


def test_penalty_at_the_longest_encoded_length_the_attention_backward_takes():
    """T' = 3914 (test_gpu_train_lengths.py's T'max of this architecture), one utterance: P."""
    _torch()
    cfg = O.make_config(**dict(BASE, dims_bidir=[128]))
    rec, _ = _run(cfg, dict(penalty_coof=COOF), B=1, T=3914, seed=81, L=11)
    assert rec.encoded_length(3914) == 3914
