"""Shared helpers for the parity tests: build a CUDA SpeechRecognizer from an oracle config."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import __graft_entry__ as graft  # noqa: E402
from oracle import lvsr_oracle as O  # noqa: E402


def package():
    return graft.load_package()


def make_recognizer(cfg, params=None, **extra):
    """A SpeechRecognizer of the oracle config `cfg` (stack_oracle's configs carry dec_stack 2); `extra` goes to the
    constructor (e.g. lm and character_map)."""
    pkg = package()
    act = {"maxout": pkg.Maxout(cfg["maxout_pieces"]), "relu": pkg.Rectifier(), "tanh": pkg.Tanh(),
           "identity": pkg.Identity()}[cfg["post_merge_activation"]]
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": cfg["num_features"]}, input_num_chars={}, eos_label=cfg["eos_label"],
        num_phonemes=cfg["num_phonemes"], dim_dec=cfg["dim_dec"], dims_bidir=cfg["dims_bidir"],
        subsample=cfg["subsample"], conv_n=cfg["conv_n"], conv_num_filters=cfg["conv_num_filters"],
        dim_matcher=cfg["dim_matcher"], post_merge_dims=cfg["post_merge_dims"], post_merge_activation=act,
        dim_output_embedding=cfg["dim_feedback"] if cfg.get("embed_outputs", True) else None,
        embed_outputs=cfg.get("embed_outputs", True), prior=cfg["prior"], energy_normalizer=cfg["energy_normalizer"],
        use_states_for_readout=cfg["use_states_for_readout"],
        max_decoded_length_scale=cfg["max_decoded_length_scale"],
        attention_type=cfg.get("attention_type", "content_and_conv"), dec_stack=cfg.get("dec_stack", 1),
        enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent, data_prepend_eos=False, **extra)
    if params is not None:
        rec.set_parameter_values(params)
    return rec


# ---- element-by-element comparison with the float64 oracle -------------------------------------------------------

def f32(a):
    """The float32 rounding of `a`, in float64: what the oracle is given so that the errors measured are the kernels'."""
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def elementwise_err(got, want, floor=0.1):
    """max |got - want| / (|want| + floor * max|want|): a wrong small element counts, a float32 absolute error of an
    element near 0 does not."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = np.abs(want).max()
    return float((np.abs(got - want) / (np.abs(want) + floor * max(scale, 1e-30))).max())


def check_weights(w, ww, errs, key="weights"):
    """Attention weights: exactly 0 where the oracle's are 0 (outside the window, masked positions, rows without a
    valid position), < 1e-29 where the oracle's are below 1e-30; errs[key] = the worst relative error per element
    elsewhere, errs[key + "_sum"] = the worst distance of a row sum from 1 over the rows with a valid position."""
    w, ww = np.asarray(w, np.float64), np.asarray(ww, np.float64)
    zero = ww == 0
    assert not np.any(w[zero]), "%s: %d non-zero weights where the oracle's are 0 (outside the window or masked)" % (
        key, int(np.count_nonzero(w[zero])))
    tiny = (ww > 0) & (ww < 1e-30)
    assert np.all(np.abs(w[tiny]) < 1e-29), key
    big = ww >= 1e-30
    errs[key] = float((np.abs(w[big] - ww[big]) / ww[big]).max()) if big.any() else 0.0
    s, sw = w.sum(-1), ww.sum(-1)
    valid = sw > 0.5                                # rows with a valid position sum to 1 in the oracle, others to 0
    assert np.all(s[~valid] == 0), key
    errs[key + "_sum"] = float(np.abs(s[valid] - 1).max()) if valid.any() else 0.0


def check_energies(e, we, errs):
    """Energies: exactly 0 outside the window; errs["energies"] = the worst absolute error over the largest magnitude."""
    e, we = np.asarray(e, np.float64), np.asarray(we, np.float64)
    assert not np.any(e[we == 0]), "non-zero energies outside the window"
    errs["energies"] = float(np.abs(e - we).max() / max(np.abs(we).max(), 1e-30))


KINK_EPS = 2e-5      # > the float32 error of a readout pre-activation on the GPU (measured <= 5e-6 at T*B = 2048)
_RO = "/recognizer/generator/readout"


def relu_readout_kinks(cfg, params, batch, eps=KINK_EPS):
    """(step, utterance, unit) of every label-unmasked row whose Rectifier readout pre-activation lies within eps of 0,
    from the float64 oracle, and the pre-activations [L, B, post_merge_dim].  [] for the other activations."""
    if cfg["post_merge_activation"] != "relu":
        return [], None
    x, m, labels, lm = batch
    out = O.recognizer_cost(cfg, params, x, m, labels, lm, return_all=True)
    pre = out["weighted_averages"] @ params[_RO + "/merge/transform_weighted_averages.W"] + params[_RO + "/post_merge/bias.b"]
    if cfg["use_states_for_readout"]:
        pre = pre + out["states"] @ params[_RO + "/merge/transform_states.W"]     # "states" = s_{i-1}, what step i reads out
    live = np.ones(labels.shape, bool) if lm is None else np.asarray(lm) > 0
    return [tuple(int(v) for v in i) for i in np.argwhere((np.abs(pre) < eps) & live[:, :, None])], pre


def _one_sided_oracle_params(cfg, params, batch):
    """The Rectifier's derivative jumps at 0.  A pre-activation within float32 error of the kink may land on either
    side of it on the GPU, so such a unit is compared with the oracle's derivative from each side: the unit's bias is
    moved so that its pre-activation is -1e-7 or +1e-7 (a change of the cost of order 1e-7 * |dcost/dx|).  Returns
    `params` first, then one parameter set per combination of sides of the units near their kink."""
    import itertools
    kinks, pre = relu_readout_kinks(cfg, params, batch)
    if not kinks:
        return [params]
    units = sorted({j for _, _, j in kinks})
    assert len(units) == len(kinks) <= 4, kinks                       # one kink per unit, few of them
    lm = batch[3]
    live = np.ones(pre.shape[:2], bool) if lm is None else np.asarray(lm) > 0
    out = [params]
    for sides in itertools.product((-1e-7, 1e-7), repeat=len(kinks)):
        p = dict(params)
        b = np.array(params[_RO + "/post_merge/bias.b"], dtype=np.float64)
        for (i, u, j), s in zip(kinks, sides):
            shift = s - pre[i, u, j]
            others = np.abs(pre[:, :, j][live])
            assert (np.sort(others)[1] > 2 * abs(shift)), (i, u, j)      # no other row of the unit crosses 0
            b[j] += shift
        p[_RO + "/post_merge/bias.b"] = b
        out.append(p)
    return out


def check_grads(cfg, params, batch, tol=1e-4, atol_frac=1e-6):
    """One lvsr_train_cost_and_grads call against the float64 gradient oracle: the cost to 1e-4, each parameter's
    gradient to `tol` of its own largest entry plus a floor of `atol_frac` of the model's largest gradient entry.  A
    Rectifier readout unit on its kink (_one_sided_oracle_params) must match the oracle from one of the two sides.
    A content-attention config (content_oracle.make_config) is compared with content_oracle's gradients."""
    if cfg.get("attention_type") == "content":
        import content_oracle as G
    else:
        from oracle import lvsr_oracle_grad as G
    pkg = package()
    rec = make_recognizer(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
    cost, grads = algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
    failures = []
    for oracle_params in _one_sided_oracle_params(cfg, params, batch):
        want_cost, want = G.cost_and_grads(cfg, oracle_params, *batch)
        gmax = max(np.abs(w).max() for w in want.values())
        errs = {}
        for k, w in want.items():
            errs[k] = float(np.abs(grads[k].astype(np.float64) - w).max() / max(np.abs(w).max(), 1e-30))
        bad = {}
        for k, e in errs.items():
            # relative to the parameter's own largest gradient entry, with a floor relative to the model's largest
            floor = atol_frac * gmax / max(np.abs(want[k]).max(), 1e-30)
            if e > tol + floor:
                bad[k] = (e, float(np.abs(want[k]).max()))
        if abs(cost - want_cost) > 1e-4 * abs(want_cost):
            bad["cost"] = (cost, want_cost)
        live = [e for k, e in errs.items() if want[k].any()]      # a zero oracle gradient is held to the floor only
        print("cost", cost, "worst rel grad err %.2e" % max(live, default=0.0), "of", len(live), "parameters")
        if not bad:
            return algo, rec
        failures.append(bad)
    raise AssertionError(failures)


def train_like_the_oracle(cfg, params, tc, steps=2, B=4, T=40):
    """`steps` process_batch calls == as many oracle train_steps (float64) on the same batches: after every step the
    cost, the gradient norm and every parameter agree.  Returns (recognizer, oracle parameters, oracle gradient norms)."""
    from collections import OrderedDict
    from oracle import lvsr_oracle_grad as G
    pkg = package()
    reg = dict(max_norm=tc["max_norm"])
    rec = make_recognizer(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(tc, reg), decay=tc["decay"])
    algo.initialize()
    ref = OrderedDict((k, v.copy()) for k, v in params.items())
    state, norms = {}, []
    for step in range(steps):
        batch = O.synthetic_batch(cfg, B=B, T=T, seed=100 + step)
        # last_cost is sequence_total_cost, the cost without the decay term (GradientDescent's docstring)
        penalty = tc["decay"] * sum(float((v ** 2).sum()) for k, v in ref.items() if G.is_weight(k))
        ref, ref_cost, ref_grads = G.train_step(cfg, ref, state, batch, tc)
        want_cost = ref_cost - penalty
        algo.process_batch(dict(zip(algo.SOURCES, batch)))
        assert abs(float(algo.last_cost.item()) - want_cost) <= 1e-4 * abs(want_cost), (step, algo.last_cost.item(), want_cost)
        norms.append(G.l2_norm(ref_grads.values()))
        assert abs(algo.total_gradient_norm() - norms[-1]) <= 1e-4 * norms[-1]
        got = rec.get_parameter_values()
        for k, v in ref.items():
            # compare the UPDATE (new - old would cancel; the parameters themselves are O(0.1..1))
            assert np.abs(got[k] - v).max() <= 2e-5 * max(1.0, np.abs(v).max()) + 1e-6, (step, k, np.abs(got[k] - v).max())
    if tc["max_norm"] > 0:
        for k, v in rec.get_parameter_values().items():
            if G.is_weight(k):
                assert (np.sqrt((v.astype(np.float64) ** 2).sum(axis=0)) <= tc["max_norm"] * (1 + 1e-5)).all(), k
    return rec, ref, norms


def rel_err(got, want):
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    return float(np.abs(got - want).max() / max(1e-12, np.abs(want).max()))


SMALL = dict(num_features=40, dims_bidir=[128], subsample=[1], dim_dec=128, conv_n=8, conv_num_filters=10,
             num_phonemes=32, post_merge_dims=[128], maxout_pieces=2)
PYRAMID = dict(num_features=40, dims_bidir=[128, 128, 128], subsample=[1, 2, 2], dim_dec=128, dim_matcher=256,
               conv_n=12, conv_num_filters=10, num_phonemes=32, post_merge_dims=[128], maxout_pieces=2)
WSJ = dict(num_features=40, dims_bidir=[256, 256, 256, 256], subsample=[1, 1, 2, 2], dim_dec=256, dim_matcher=512,
           conv_n=100, conv_num_filters=10, num_phonemes=32, post_merge_dims=[256], maxout_pieces=2)


_READOUT = "/recognizer/generator/readout/post_merge/mlp/linear_0"


def bottom_recognizer(cfg, params=None, lm=None, cmap=None):
    """A SpeechRecognizer of a bottom_oracle config (a bottom MLP in front of the encoder; forward-only encoder layers
    when the config has bidir False)."""
    pkg = package()
    content = cfg.get("attention_type") == "content"
    act = {"relu": pkg.Rectifier(), "tanh": pkg.Tanh()}[cfg["bottom"]["activation"]]
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": cfg["num_features"]}, input_num_chars={}, eos_label=cfg["eos_label"],
        num_phonemes=cfg["num_phonemes"], dim_dec=cfg["dim_dec"], dims_bidir=cfg["dims_bidir"],
        subsample=cfg["subsample"], conv_n=None if content else cfg["conv_n"],
        conv_num_filters=cfg["conv_num_filters"], dim_matcher=cfg["dim_matcher"],
        post_merge_dims=cfg["post_merge_dims"], post_merge_activation=pkg.Maxout(cfg["maxout_pieces"]),
        dim_output_embedding=cfg["dim_feedback"] if cfg.get("embed_outputs", True) else None,
        embed_outputs=cfg.get("embed_outputs", True), prior=None if content else cfg["prior"],
        energy_normalizer=None if content else cfg["energy_normalizer"],
        attention_type="content" if content else "content_and_conv",
        max_decoded_length_scale=cfg["max_decoded_length_scale"], enc_transition=pkg.GatedRecurrent,
        dec_transition=pkg.GatedRecurrent, data_prepend_eos=False, lm=lm, character_map=cmap,
        dec_stack=cfg.get("dec_stack", 1), bottom=dict(dims=cfg["bottom"]["dims"], activation=act),
        bidir=cfg.get("bidir", True))
    if params is not None:
        rec.set_parameter_values(params)
    return rec


def bottom_params(cfg, seed, gain=1.0, eos_bias=None):
    """Trained-like float32 parameters (scale 10) with biases of the bottom drawn too."""
    import bottom_oracle
    from collections import OrderedDict
    p = bottom_oracle.init_params(cfg, seed=seed, scale=10.0)
    rng = np.random.RandomState(seed + 100)
    for i, d in enumerate(cfg["bottom"]["dims"]):
        p[bottom_oracle.linear_name(i) + ".W"] *= 10.0 / np.sqrt(p[bottom_oracle.linear_name(i) + ".W"].shape[0])   # pre-activations O(1)
        p[bottom_oracle.linear_name(i) + ".b"] = rng.normal(0, 0.3, size=d)
    p[_READOUT + ".W"] = p[_READOUT + ".W"] * gain
    if eos_bias is not None:
        p[_READOUT + ".b"][cfg["eos_label"]] = eos_bias
    return OrderedDict((k, f32(v)) for k, v in p.items())


INT_MAX = 2 ** 31 - 1


def check_overlap_claims(rec, plan, B, subsample, ndir=2):
    """Every tile the launch beside a scan claimed had all its rows final at the progress it was claimed at: input frame
    f of layer l is the scan's output frame f, stored at scan step f k by the forward direction and at step T - 1 - f k
    by the backward one, so it is final once forward progress > f k and backward progress >= T - f k.  A forward-only
    scan (ndir 1) has no backward progress: its records must hold INT_MAX there, and only the forward rule decides."""
    for l, p in enumerate(plan):
        if not p["overlap"]:
            continue
        T, k, M = plan[l - 1]["T"], subsample[l - 1], p["T"] * B
        tiles = p["tiles_beside"] + p["tiles_after"]
        rec_ = rec.encoder_overlap_claims(l, tiles).astype(np.int64)
        rec_ = rec_[rec_[:, 0] > 0]
        assert len(rec_) == p["tiles_beside"], (l, len(rec_), p)
        r0 = (rec_[:, 0] - 1) * 128
        r1 = np.minimum(r0 + 128, M) - 1
        f_lo, f_hi = r0 // B, r1 // B
        if ndir == 1:
            assert (rec_[:, 2] == INT_MAX).all(), ("layer %d: backward progress recorded beside a forward-only scan" % l,
                                                   rec_[rec_[:, 2] != INT_MAX][:5])
            early = rec_[:, 1] < f_hi * k + 1
        else:
            early = (rec_[:, 1] < f_hi * k + 1) | (rec_[:, 2] < T - f_lo * k)
        assert not early.any(), ("layer %d: %d of %d tiles claimed before their rows were final" %
                                 (l, early.sum(), len(rec_)), rec_[early][:5], f_lo[early][:5], f_hi[early][:5])


def stream_mid(T, k, B, tiles_m, ndir):
    """gemm_tc.cu gemm_f16_stream: the m-tile whose rows become final first.  Output frame f is the scan's step f k:
    final after f k + 1 forward steps and, with two directions, T - f k backward steps; mid is the m-tile of the first
    frame with the fewest steps max(both) (two directions) or f k + 1 (forward only: frame 0)."""
    best, fmid = None, 0
    for f in range(-(-T // k)):
        ready = f * k + 1 if ndir == 1 else max(f * k + 1, T - f * k)
        if best is None or ready < best:
            best, fmid = ready, f
    return min(fmid * B // 128, tiles_m - 1)


def stream_m_tile(i, mid, tiles_m):
    """gemm_tc.cu stream_m_tile: claim index i (in whole m-tiles) -> m-tile: mid, then alternately one further right
    and one further left, then the rest of the longer side."""
    if i == 0:
        return mid
    j, left, right = i - 1, mid, tiles_m - 1 - mid
    both = min(left, right)
    if j < 2 * both:
        return mid - 1 - (j >> 1) if j & 1 else mid + 1 + (j >> 1)
    return mid + 1 + j - both if right > left else mid - 1 - (j - both)


def check_overlap_claim_order(rec, plan, B, subsample, widths, ndir):
    """Claim c beside the scan took m-tile stream_m_tile(c // tiles_n, mid, tiles_m), with tiles_n = ndir 3 D / 128
    column tiles of the fork projection and mid = stream_mid's.  Returns {layer: (mid, tiles beside)}."""
    out = {}
    for l, p in enumerate(plan):
        if not p["overlap"] or not p["tiles_beside"]:
            continue
        T, k, M = plan[l - 1]["T"], subsample[l - 1], p["T"] * B
        tiles_m, tiles_n = -(-M // 128), ndir * 3 * widths[l] // 128
        mid = stream_mid(T, k, B, tiles_m, ndir)
        recs = rec.encoder_overlap_claims(l, p["tiles_beside"] + p["tiles_after"]).astype(np.int64)
        c = np.flatnonzero(recs[:, 0] > 0)
        assert np.array_equal(c, np.arange(p["tiles_beside"])), (l, c[:8], p)
        want = np.array([stream_m_tile(i // tiles_n, mid, tiles_m) for i in c])
        got = recs[c, 0] - 1
        bad = np.flatnonzero(got != want)
        assert not bad.size, ("layer %d: %d of %d claims out of order (mid %d of %d m-tiles)" %
                              (l, bad.size, c.size, mid, tiles_m), c[bad][:5], got[bad][:5], want[bad][:5])
        out[l] = (mid, int(c.size))
    return out


def check_unidirectional_grads(cfg, params, batch, tol=1e-4, atol_frac=1e-6):
    """check_grads' comparison for a forward-only model (net.bidir: False) against the gradient oracle of
    tests/unidirectional_oracle.py; returns the recognizer."""
    import unidirectional_oracle as U
    pkg = package()
    rec = make_recognizer(cfg, params, bidir=False)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
    cost, grads = algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
    want_cost, want = U.cost_and_grads(cfg, params, *batch)
    assert set(grads) == set(want)
    gmax = max(np.abs(w).max() for w in want.values())
    bad = {}
    worst = 0.0
    for k, w in want.items():
        e = float(np.abs(grads[k].astype(np.float64) - w).max() / max(np.abs(w).max(), 1e-30))
        floor = atol_frac * gmax / max(np.abs(w).max(), 1e-30)
        if w.any():
            worst = max(worst, e)
        if e > tol + floor:
            bad[k] = e
    print("cost", cost, want_cost, "worst rel grad err %.2e" % worst)
    assert abs(cost - want_cost) <= 1e-4 * abs(want_cost), (cost, want_cost)
    assert not bad, bad
    return rec


def bench_recognizer():
    """The recognizer bench.py --mode train builds (bench.NET at bench.TRAIN_WORKLOAD's features and vocabulary)."""
    import bench
    pkg = package()
    W, N = bench.TRAIN_WORKLOAD, bench.NET
    return pkg.SpeechRecognizer(
        input_dims={"recordings": W["F"]}, input_num_chars={}, eos_label=W["V"] - 1, num_phonemes=W["V"],
        dim_dec=N["dim_dec"], dims_bidir=N["dims_bidir"], subsample=N["subsample"], conv_n=N["conv_n"],
        conv_num_filters=N["conv_num_filters"], dim_matcher=N["dim_matcher"], post_merge_dims=N["post_merge_dims"],
        post_merge_activation=pkg.Maxout(2), enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent)
