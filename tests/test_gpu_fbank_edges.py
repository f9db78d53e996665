"""The filterbank front end (csrc/fbank.cu) at every option and signal edge it accepts.

Each stage is compared at its own precision, so that a weak mel bin's round-off does not hide an error elsewhere:
  * static columns (log energy, log mel bins) against the float64 oracle and, where tests/golden/fbank_kaldi_golden.npz
    holds the same options and signal, against torchaudio's features directly: linear mel energies relative to the
    frame's peak (LIN_TOL), logs absolutely where the energy is at least 1e-4 of the peak and for the log energy
    (LOG_TOL); a value the oracle floors must be float32 log(FLT_EPSILON) to 1 ulp;
  * delta columns against the oracle's add_deltas of the GPU's own static columns, within the float32 bound of the
    tap sum: (taps + 2) u sum_k |s_k| |x_{t+k}| (u = 2^-24: the float32 rounding of each scale, then one rounding per
    fused multiply-add of the chain);
  * CMVN against the oracle's ApplyCmvn of the GPU's own features, within 3 u (|x scale| + |offset|) (the float32
    scale and offset, then the fused multiply-add), and its stats against float64 sums of those features;
  * frames past an utterance's end: exactly 0, mask 0.
Measured worsts over this file on an H100 80GB HBM3 (700 W): linear 2.0e-6, log 1.7e-5, deltas 0.23 of their bound,
CMVN 0.63 of its bound, dithered features (FEAT_TOL) 1.3e-4; the large DC offset stays inside its derived bound and
within 1.6e-3 of torchaudio.
"""
import numpy as np
import pytest

import fbank_helpers as H
import fbank_oracle as F
from helpers import package

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
RECORDS = {r["name"]: r for r in H.load_golden()}

# options torchaudio's fbank has no counterpart for: deltas of every order and window
DELTA_CASES = {"order_1_window_1": dict(delta_order=1, delta_window=1), "order_1": dict(delta_order=1),
               "order_2_window_3": dict(delta_window=3), "order_3": dict(delta_order=3),
               "order_3_window_4": dict(delta_order=3, delta_window=4)}
OPTION_CASES = dict([(n, r["options"]) for n, r in RECORDS.items() if r["signal"] == "tones"] +
                    list(DELTA_CASES.items()))
EDGE_CASES = [n for n, r in RECORDS.items() if r["signal"] not in ("tones", "dc_noise")]


def _ulp_floor(got):
    return np.abs(got.astype(np.float32) - H.LOG_EPS32) <= np.spacing(np.abs(H.LOG_EPS32))


def _static(got, x, o, errs, golden=None):
    """GPU static columns got [n, D0] of utterance x against the oracle (and torchaudio's `golden` record)."""
    st, lin = F.fbank(x, o, linear=True)
    ne = int(o["use_energy"])
    floored = lin <= F.FLT_EPSILON
    assert _ulp_floor(got[:, ne:][floored]).all(), "a floored mel bin"
    live = ~floored.all(1)                                       # frames with any energy
    if live.any():
        H.static_errors(got[live], st[live], np.where(floored, 0.0, lin)[live], ne, errs)
    if ne:
        errs["log"] = max(errs.get("log", 0.0), float(np.abs(got[:, 0] - st[:, 0]).max()))
    if golden is not None:
        want = golden["feats"]
        if want.dtype == np.float32:                             # the float32 floor records
            at = want == H.LOG_EPS32
            assert _ulp_floor(got[at]).all(), "torchaudio's floor"
        elif live.all():
            H.static_errors(got, want, np.exp(want[:, ne:]), ne, errs)
    assert errs.get("lin", 0.0) <= H.LIN_TOL and errs.get("log", 0.0) <= H.LOG_TOL, errs


def _delta_bound(x, order, window):
    """[T, D0 order]: (taps + 2) u sum_k |s_k| |x_clamp(t+k)| for each order."""
    x = np.abs(np.asarray(x, np.float64))
    T = x.shape[0]
    out = []
    for i, sc in enumerate(F.delta_scales(order, window)[1:], start=1):
        reach = i * window
        acc = np.zeros_like(x)
        for j in range(-reach, reach + 1):
            acc += abs(sc[j + reach]) * x[np.clip(np.arange(T) + j, 0, T - 1)]
        out.append((2 * reach + 3) * U * acc)
    return np.concatenate(out, axis=1)


def _deltas(feats, n, b, o, errs):
    """The delta columns of utterance row b (n frames) against add_deltas of its own static columns."""
    D0 = o["num_mel_bins"] + o["use_energy"]
    if o["delta_order"] == 0:
        return
    st = feats[:n, b, :D0]
    want = F.add_deltas(st, o["delta_order"], o["delta_window"])[:, D0:]
    err = np.abs(feats[:n, b, D0:] - want)
    bound = _delta_bound(st, o["delta_order"], o["delta_window"])
    errs["delta"] = max(errs.get("delta", 0.0), float((err / bound).max()))
    assert (err <= bound).all(), ("deltas", float((err - bound).max()))


def _stages(fb, o, wavs, feats, mask, goldens=None):
    """Mask, padding, static columns and deltas of a batch; returns the worst errors."""
    feats, mask = feats.cpu().numpy().astype(np.float64), mask.cpu().numpy()
    frames = [F.num_frames(len(x), o) for x in wavs]
    assert [fb.num_frames(len(x)) for x in wavs] == frames
    assert np.array_equal(mask, (np.arange(feats.shape[0])[:, None] < np.array(frames)[None, :]).astype(np.float32))
    assert not feats[mask == 0].any(), "padded frames must be exactly 0"
    errs = {}
    D0 = o["num_mel_bins"] + o["use_energy"]
    for b, x in enumerate(wavs):
        _static(feats[:frames[b], b, :D0], x, o, errs, None if goldens is None else goldens[b])
        _deltas(feats, frames[b], b, o, errs)
    return errs


def _cmvn_bound(x, stats):
    D = stats.shape[1] - 1
    n = stats[0, D]
    mean = stats[0, :D] / n
    scale = 1.0 / np.sqrt(np.maximum(stats[1, :D] / n - mean ** 2, 1e-20))
    return 3 * U * (np.abs(x * scale) + np.abs(mean * scale)) + 1e-30


def _cmvn(fb, o, wavs, feats, mask, errs):
    """Stats of the GPU's features against float64 sums; compute(cmvn=) and apply() against ApplyCmvn of them."""
    torch = H.torch_or_skip()
    f64, m = feats.cpu().numpy().astype(np.float64), mask.cpu().numpy()
    cmvn = package().GlobalCmvn(fb)
    cmvn.accumulate(feats, mask)
    want = F.cmvn_stats([f64[:int(m[:, b].sum()), b] for b in range(f64.shape[1])])
    np.testing.assert_allclose(cmvn.stats, want, rtol=1e-12, atol=1e-12 * np.abs(want).max())
    normed, nm = fb.compute(wavs, cmvn=cmvn.stats, T=feats.shape[0])
    assert torch.equal(nm, mask)
    ref = np.where(m[..., None] > 0, F.apply_cmvn(f64, cmvn.stats), 0.0)
    err = np.abs(normed.cpu().numpy() - ref)
    bound = _cmvn_bound(f64, cmvn.stats)
    errs["cmvn"] = max(errs.get("cmvn", 0.0), float((err / bound).max()))
    assert (err <= bound).all(), ("cmvn", float((err - bound).max()))
    assert torch.equal(cmvn.apply(feats.clone(), mask), normed)


@pytest.mark.parametrize("cmvn", [False, True], ids=["raw", "cmvn"])
@pytest.mark.parametrize("name", sorted(OPTION_CASES))
def test_option_matrix(name, cmvn):
    """Every accepted option: the torchaudio record's utterance and two more, of 17 frames and of one frame."""
    H.torch_or_skip()
    fb, o = H.make_fb(dither=0.0, **OPTION_CASES[name])
    W, S, _ = F.frame_sizes(o)
    rng = np.random.RandomState(len(name))
    rec = RECORDS.get(name)
    first = rec["wave"] if rec else H.edge_signal("tones", o)
    wavs = [first] + H.waves(rng, [W + 16 * S + S // 2, W], o["sample_frequency"])
    assert fb.feature_dim == (o["num_mel_bins"] + o["use_energy"]) * (o["delta_order"] + 1)
    feats, mask = fb.compute(wavs)
    errs = _stages(fb, o, wavs, feats, mask, [rec, None, None])
    if cmvn:
        _cmvn(fb, o, wavs, feats, mask, errs)
    print(name, errs)


@pytest.mark.parametrize("name", EDGE_CASES)
def test_edge_signals(name):
    """Silence, silent frames inside a loud utterance, DC, full scale, Nyquist, tones on FFT and mel bin centres and
    impulses at a frame's first and last samples and at a shift boundary, beside a loud utterance."""
    H.torch_or_skip()
    rec = RECORDS[name]
    fb, o = H.make_fb(dither=0.0, **rec["options"])
    wavs = [rec["wave"], H.edge_signal("tones", o, frames=20)]
    feats, mask = fb.compute(wavs, T=22)
    print(name, _stages(fb, o, wavs, feats, mask, [rec, None]))


@pytest.mark.parametrize("raw_energy", [True, False])
def test_digital_silence(raw_energy):
    """Every static column is float32 log(FLT_EPSILON) to 1 ulp, under either energy.  The deltas are the float32
    tap sums of a constant column: not exactly 0, because the float32 scales do not sum to exactly 0 (as in Kaldi's
    float add-deltas), but within the tap-sum bound of 0."""
    H.torch_or_skip()
    fb, o = H.make_fb(dither=0.0, raw_energy=raw_energy, delta_order=3, delta_window=4)
    wavs = [np.zeros(400 + 40 * 160, np.int16), np.zeros(400, np.int16)]
    feats, mask = fb.compute(wavs, T=45)
    f = feats.cpu().numpy()
    for b, n in enumerate((41, 1)):
        assert _ulp_floor(f[:n, b, :41]).all()
        bound = _delta_bound(f[:n, b, :41], 3, 4)
        assert (np.abs(f[:n, b, 41:]) <= bound).all()
    assert not f[41:, 0].any() and not f[1:, 1].any()


def test_large_dc_offset_under_small_noise():
    """20000 + N(0, 2): the frame mean cancels in float32.  The kernel sums a frame's W samples as per-lane sequential
    sums of up to 4 ceil(ceil(W / 4) / 32) samples and a 5-level shuffle tree, so the float32 sum is off by at most
    n u sum|x| with n = 4 ceil(ceil(W / 4) / 32) + 5 additions, and the division by W adds u |mean|: the mean is off
    by at most delta = (n + 1) u sum|x| / W (0.025 for W = 400 here).  The samples are integers near the mean, so
    x - mean is exact (Sterbenz) and every DC-free sample carries the same offset e, |e| <= delta.  The bound of a
    static column is then the oracle's change when the frame mean moves by +-delta (each column is monotone in e on
    either side of its extremum, so the two ends bound it) plus the usual LIN_TOL / LOG_TOL."""
    H.torch_or_skip()
    rec = RECORDS["dc_noise"]
    fb, o = H.make_fb(dither=0.0, delta_order=0)
    x = rec["wave"].astype(np.float64)
    feats, _ = fb.compute([rec["wave"]])
    got = feats.cpu().numpy().astype(np.float64)[:, 0]
    W, S, _ = F.frame_sizes(o)
    n = 4 * (((W + 3) // 4 + 31) // 32) + 5
    flat = F.options(**dict(o, remove_dc_offset=False))
    worst = 0.0
    for t in range(got.shape[0]):
        fr = x[t * S:t * S + W]
        delta = (n + 1) * U * np.abs(fr).sum() / W
        moved = [F.fbank(fr - fr.mean() - e, flat, linear=True) for e in (0.0, -delta, delta)]
        (st0, lin0), ends = moved[0], moved[1:]
        dlog = np.max([np.abs(st - st0) for st, _ in ends], axis=0)[0]
        dlin = np.max([np.abs(lin - lin0) for _, lin in ends], axis=0)[0]
        peak = lin0.max()
        assert (np.abs(np.exp(got[t, 1:]) - lin0[0]) <= dlin + H.LIN_TOL * peak).all(), t
        strong = lin0[0] >= 1e-4 * peak
        assert (np.abs(got[t, 1:] - st0[0, 1:])[strong] <= dlog[1:][strong] + H.LOG_TOL).all(), t
        assert abs(got[t, 0] - st0[0, 0]) <= dlog[0] + H.LOG_TOL, t
        worst = max(worst, float(np.abs(got[t] - rec["feats"][t]).max()))
    print("dc_noise worst |gpu - torchaudio|", worst)


def test_fft_below_eight_points_is_refused():
    """P = 8 is the smallest FFT the mel-bin check accepts (W5_P8 and W8_P8 run in test_option_matrix): at P = 4 the
    only FFT bin above 0 Hz cannot fill 3 mel bins."""
    H.torch_or_skip()
    for lo in (0.0, 20.0, 1000.0):
        o = F.options(frame_length=0.25, frame_shift=0.25, low_freq=lo, num_mel_bins=3)
        assert F.frame_sizes(o) == (4, 4, 4)
        empty = int(np.flatnonzero(~(F.mel_banks(o) > 0).any(1))[0])
        with pytest.raises(RuntimeError, match="mel bin %d has no FFT bin" % empty):
            H.make_fb(**o)


@pytest.mark.parametrize("fs", [16000.0, 8000.0])
def test_num_mel_bins_limits(fs):
    """3 bins and the largest count whose every bin holds an FFT bin run; one more is refused naming its empty bin."""
    torch = H.torch_or_skip()
    nb = 3
    while (F.mel_banks(F.options(sample_frequency=fs, num_mel_bins=nb + 1))[:, :-1] > 0).any(1).all():
        nb += 1
    assert nb == {16000.0: 126, 8000.0: 95}[fs]                # the records test_option_matrix runs
    o = F.options(sample_frequency=fs, num_mel_bins=nb + 1)
    empty = int(np.flatnonzero(~(F.mel_banks(o) > 0).any(1))[0])
    with pytest.raises(RuntimeError, match="num_mel_bins %d too large: mel bin %d has no FFT bin" % (nb + 1, empty)):
        H.make_fb(**o)
    fb, o = H.make_fb(dither=0.0, sample_frequency=fs, num_mel_bins=3)
    wavs = H.waves(np.random.RandomState(3), [int(fs), 1000], fs)
    feats, mask = fb.compute(wavs)
    assert torch.isfinite(feats).all()
    print(fs, nb, _stages(fb, o, wavs, feats, mask))


def test_frame_shift_limits():
    """S = 1 sample and S > W run in test_option_matrix.  The shared-memory check admits a run of 16 frames while
    4 (8 warps x 2 x 512 + W rounded to 4 + P + 15 S + W + 8) bytes fit in 226 KB: at 16 kHz S <= 3222 samples, so
    201 ms (3216) runs on the GPU and 202 ms is refused."""
    H.torch_or_skip()
    W, P = 400, 512
    limit = (226 * 1024 // 4 - (8 * 2 * 512 + W + P + W + 8)) // 15
    assert limit == 3222 and int(16 * 201.0) <= limit < int(16 * 202.0)
    with pytest.raises(RuntimeError, match=r"frame_shift 202 ms \(3232 samples\) is too long for a run of 16 frames"):
        H.make_fb(frame_shift=202.0)
    fb, o = H.make_fb(dither=0.0, frame_shift=201.0)
    wavs = H.waves(np.random.RandomState(4), [W + 17 * 3216, W + 3216 - 1], 16000.0)
    feats, mask = fb.compute(wavs)
    assert feats.shape[0] == 18
    print(_stages(fb, o, wavs, feats, mask))


@pytest.mark.parametrize("window", [1, 2, 3, 4])
@pytest.mark.parametrize("order", [1, 2, 3])
def test_deltas_in_isolation(order, window):
    """Utterances of 1, 2, reach, reach + 1, 2 reach + 1 and 300 frames in one ragged batch, T past the longest."""
    H.torch_or_skip()
    fb, o = H.make_fb(dither=0.0, delta_order=order, delta_window=window)
    reach = order * window
    frames = [1, 2, reach, reach + 1, 2 * reach + 1, 300]
    wavs = H.waves(np.random.RandomState(10 * order + window), [400 + (n - 1) * 160 + 37 for n in frames])
    feats, mask = fb.compute(wavs, T=305)
    f = feats.cpu().numpy().astype(np.float64)
    errs = {}
    for b, n in enumerate(frames):
        _deltas(f, n, b, o, errs)
    assert not f[np.arange(305)[:, None] >= np.array(frames)[None, :]].any()
    print(order, window, errs)


def test_batch_layout_at_run_boundaries():
    """Frame counts 15, 16, 17, 31, 32 and 33 (the 16-frame runs' edges) in one batch, given as a list, as a tensor
    whose row stride is the longest length rounded up to 4, and with T past every utterance."""
    torch = H.torch_or_skip()
    fb, o = H.make_fb(dither=0.0)
    frames = [15, 16, 17, 31, 32, 33]
    lengths = [400 + (n - 1) * 160 + k for n, k in zip(frames, (0, 159, 1, 3, 0, 2))]
    wavs = H.waves(np.random.RandomState(5), lengths)
    stride = (max(lengths) + 3) // 4 * 4
    x = torch.zeros((len(wavs), stride), dtype=torch.float32, device="cuda")
    for b, w in enumerate(wavs):
        x[b, :len(w)] = torch.as_tensor(w.astype(np.float32))
    a, am = fb.compute(wavs)
    b_, bm = fb.compute(x, lengths=lengths)
    assert a.shape[0] == 33 and torch.equal(a, b_) and torch.equal(am, bm)
    c, cm = fb.compute(wavs, T=50)
    assert torch.equal(c[:33], a) and torch.equal(cm[:33], am) and not c[33:].any() and not cm[33:].any()
    print(_stages(fb, o, wavs, c, cm))


@pytest.mark.parametrize("rows", [1, 263, 264, 265, 527, 529, 791, 793])
def test_cmvn_wide_at_chunk_boundaries(rows):
    """Delta order 3 with 80 bins (324 columns, more than the kernels' 256 threads), at row counts around the
    accumulation's 264 partial sums, with a mask and with mask=None."""
    torch = H.torch_or_skip()
    fb, o = H.make_fb(dither=0.0, num_mel_bins=80, delta_order=3)
    D = fb.feature_dim
    assert D == 324
    T = {1: 1, 263: 263, 264: 132, 265: 53, 527: 527, 529: 529, 791: 113, 793: 793}[rows]
    B = rows // T
    rng = np.random.RandomState(rows)
    x = (rng.normal(0, 1, size=(T, B, D)) * rng.uniform(0.1, 30, size=D) + rng.normal(0, 20, size=D)).astype(np.float32)
    m = (rng.uniform(size=(T, B)) < 0.8).astype(np.float32)
    m[0, 0] = 1
    xs, ms = torch.as_tensor(x, device="cuda"), torch.as_tensor(m, device="cuda")
    x64 = x.astype(np.float64).reshape(rows, D)
    errs = {}
    for mask, keep in ((ms, m.reshape(rows) > 0), (None, np.ones(rows, bool))):
        cmvn = package().GlobalCmvn(fb)
        cmvn.accumulate(xs, mask)
        want = F.cmvn_stats([x64[keep]])
        np.testing.assert_allclose(cmvn.stats, want, rtol=1e-12, atol=1e-12 * np.abs(want).max())
        got = cmvn.apply(xs.clone(), mask).cpu().numpy().astype(np.float64).reshape(rows, D)
        ref = np.where(keep[:, None], F.apply_cmvn(x64, cmvn.stats), x64)
        bound = _cmvn_bound(x64, cmvn.stats)
        errs["cmvn"] = max(errs.get("cmvn", 0.0), float((np.abs(got - ref) / bound).max()))
        assert (np.abs(got - ref) <= bound).all()
    # the same stats applied inside compute(), over 324 columns
    wavs = H.waves(rng, [400 + 40 * 160, 1000])
    feats, mask = fb.compute(wavs)
    _cmvn(fb, o, wavs, feats, mask, errs)
    print(rows, errs)


def test_cmvn_refused_until_it_has_frames():
    """A GlobalCmvn with no frames would normalise by 0 / 0: it is refused until accumulate or stats = has run."""
    torch = H.torch_or_skip()
    pkg = package()
    fb, o = H.make_fb(dither=0.0, delta_order=0)
    wavs = H.waves(np.random.RandomState(6), [4000, 1000])
    feats, mask = fb.compute(wavs)
    cmvn = pkg.GlobalCmvn(fb)
    with pytest.raises(ValueError, match="no frames"):
        cmvn.apply(feats.clone(), mask)
    with pytest.raises(ValueError, match="no frames"):
        fb.compute(wavs, cmvn=cmvn)
    cmvn.stats = np.zeros((2, 42))
    with pytest.raises(ValueError, match="no frames"):
        cmvn.apply(feats.clone(), mask)
    cmvn.accumulate(feats, mask)
    normed = cmvn.apply(feats.clone(), mask)
    assert torch.isfinite(normed).all()
    loaded = pkg.GlobalCmvn(fb, cmvn.stats)
    assert torch.equal(fb.compute(wavs, cmvn=loaded)[0], normed)


@pytest.mark.parametrize("dither", [0.5, 4.0])
def test_dither_replay(dither):
    H.torch_or_skip()
    fb, o = H.make_fb(dither=dither, seed=11)
    wavs = H.waves(np.random.RandomState(7), [5000, 400, 3210])
    feats, mask = fb.compute(wavs)
    draws = fb.dither_sample(len(wavs), feats.shape[0]).cpu().numpy()
    print(dither, H.check(feats, mask, wavs, o, draws=list(draws)))


def test_seed_uses_both_halves():
    torch = H.torch_or_skip()
    wavs = H.waves(np.random.RandomState(8), [4000, 2000])
    s = 12345
    lo, _ = H.make_fb(dither=1.0, seed=s)
    hi, _ = H.make_fb(dither=1.0, seed=s + 2 ** 32)
    assert not torch.equal(lo.compute(wavs)[0], hi.compute(wavs)[0])
    assert not torch.equal(lo.dither_sample(2, 20), hi.dither_sample(2, 20))
