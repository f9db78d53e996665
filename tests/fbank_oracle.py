"""Float64 restatement of the recipes' features: Kaldi's compute-fbank-feats, add-deltas and global CMVN
(exp/wsj/write_hdf_dataset.sh:94-105), written from their definition (DESIGN §1 (j)), not from Kaldi's source.

Samples are in int16 units, one utterance per 1-D array.  The dither is not drawn here: a test passes the draws the
GPU used (lvsr_frontend_dither_sample) as `draws` [frames, W], scaled by `dither`.
"""
import numpy as np

FLT_EPSILON = float(np.finfo(np.float32).eps)       # floor of the log energy (raw or windowed) and of the mel energies

DEFAULTS = dict(sample_frequency=16000.0, frame_length=25.0, frame_shift=10.0, dither=1.0, remove_dc_offset=True,
                preemphasis_coefficient=0.97, window_type="povey", round_to_power_of_two=True, snip_edges=True,
                num_mel_bins=40, low_freq=20.0, high_freq=0.0, use_energy=True, raw_energy=True, energy_floor=0.0,
                use_log_fbank=True, use_power=True, htk_compat=False, delta_order=2, delta_window=2)


def options(**kw):
    o = dict(DEFAULTS)
    o.update(kw)
    return o


def frame_sizes(o):
    """(W, S, P): frame length, shift and padded FFT length in samples."""
    fs = o["sample_frequency"]
    W, S = int(fs * 0.001 * o["frame_length"]), int(fs * 0.001 * o["frame_shift"])
    P = 1
    while P < W:
        P *= 2
    return W, S, (P if o["round_to_power_of_two"] else W)


def num_frames(N, o):
    W, S, _ = frame_sizes(o)
    return 0 if N < W else 1 + (N - W) // S


def window(o):
    W = frame_sizes(o)[0]
    a = 2 * np.pi * np.arange(W) / (W - 1)
    return {"povey": (0.5 - 0.5 * np.cos(a)) ** 0.85, "hamming": 0.54 - 0.46 * np.cos(a),
            "hanning": 0.5 - 0.5 * np.cos(a), "rectangular": np.ones(W)}[o["window_type"]]


def mel(f):
    return 1127.0 * np.log(1.0 + np.asarray(f, np.float64) / 700.0)


def inverse_mel(m):
    return 700.0 * (np.exp(np.asarray(m, np.float64) / 1127.0) - 1.0)


def mel_edges(o):
    """[num_mel_bins, 3] (left, centre, right) of every bin, in mel."""
    fs, n = o["sample_frequency"], o["num_mel_bins"]
    hi = o["high_freq"] if o["high_freq"] > 0 else 0.5 * fs + o["high_freq"]
    lo_m, hi_m = mel(o["low_freq"]), mel(hi)
    d = (hi_m - lo_m) / (n + 1)
    b = np.arange(n)[:, None] + np.arange(3)[None, :]
    return lo_m + b * d


def triangle(m, edges):
    """Weights of mel values m [K] in bins edges [n, 3] -> [n, K]: (m - left) / (centre - left) up to the centre,
    (right - m) / (right - centre) above it, 0 outside the open interval (left, right)."""
    left, centre, right = (edges[:, k:k + 1] for k in range(3))
    m = np.asarray(m, np.float64)[None, :]
    up = (m - left) / (centre - left)
    down = (right - m) / (right - centre)
    return np.where((m > left) & (m < right), np.where(m <= centre, up, down), 0.0)


def mel_banks(o):
    """[num_mel_bins, P/2 + 1] weights over the power spectrum; the Nyquist column is 0."""
    fs = o["sample_frequency"]
    P = frame_sizes(o)[2]
    f = np.arange(P // 2) * fs / P
    w = triangle(mel(f), mel_edges(o))
    return np.concatenate([w, np.zeros((w.shape[0], 1))], axis=1)


def process_frames(x, o, draws=None):
    """Per frame of utterance x [N]: (windowed frame [T, W], power spectrum [T, P/2 + 1], log energy [T])."""
    W, S, P = frame_sizes(o)
    T = num_frames(len(x), o)
    idx = np.arange(T)[:, None] * S + np.arange(W)[None, :]
    fr = np.asarray(x, np.float64)[idx]
    if draws is not None and o["dither"] != 0:
        fr = fr + o["dither"] * np.asarray(draws, np.float64)[:T, :W]
    if o["remove_dc_offset"]:
        fr = fr - fr.mean(axis=1, keepdims=True)
    if o["raw_energy"]:
        log_e = np.log(np.maximum((fr ** 2).sum(1), FLT_EPSILON))
    p = o["preemphasis_coefficient"]
    pre = fr.copy()
    pre[:, 1:] -= p * fr[:, :-1]
    pre[:, 0] -= p * fr[:, 0]
    win = pre * window(o)[None, :]
    if not o["raw_energy"]:
        log_e = np.log(np.maximum((win ** 2).sum(1), FLT_EPSILON))
    spec = np.abs(np.fft.rfft(win, n=P, axis=1)) ** 2
    if not o["use_power"]:
        spec = np.sqrt(spec)
    return win, spec, log_e


def fbank(x, o, draws=None, linear=False):
    """compute-fbank-feats of one utterance -> [T, D0] ([log energy, bins] with use_energy); linear=True also returns
    the mel energies before the log [T, num_mel_bins]."""
    _, spec, log_e = process_frames(x, o, draws)
    energies = spec @ mel_banks(o).T
    feats = np.log(np.maximum(energies, FLT_EPSILON))
    if o["use_energy"]:
        if o["energy_floor"] > 0:
            log_e = np.maximum(log_e, np.log(o["energy_floor"]))
        feats = np.concatenate([log_e[:, None], feats], axis=1)
    return (feats, energies) if linear else feats


def delta_scales(order, window):
    """add-deltas: scales_0 = [1], scales_i = conv(scales_{i-1}, [-w .. w]) / sum j^2."""
    out = [np.ones(1)]
    k = np.arange(-window, window + 1, dtype=np.float64)
    for _ in range(order):
        out.append(np.convolve(out[-1], k) / (k ** 2).sum())
    return out


def add_deltas(x, order=2, window=2):
    """[T, D0] -> [T, D0 (order + 1)] with frame indices clamped to [0, T-1]."""
    x = np.asarray(x, np.float64)
    T = x.shape[0]
    cols = [x]
    for i, sc in enumerate(delta_scales(order, window)[1:], start=1):
        reach = i * window
        acc = np.zeros_like(x)
        for j in range(-reach, reach + 1):
            acc += sc[j + reach] * x[np.clip(np.arange(T) + j, 0, T - 1)]
        cols.append(acc)
    return np.concatenate(cols, axis=1)


def features(x, o, draws=None):
    """fbank | add-deltas of one utterance -> [T, D]."""
    f = fbank(x, o, draws)
    return add_deltas(f, o["delta_order"], o["delta_window"]) if o["delta_order"] > 0 else f


def cmvn_stats(feature_list):
    """Kaldi's global stats [2, D+1]: column sums | frame count, sums of squares | 0."""
    D = feature_list[0].shape[1]
    s = np.zeros((2, D + 1))
    for f in feature_list:
        f = np.asarray(f, np.float64)
        s[0, :D] += f.sum(0)
        s[1, :D] += (f ** 2).sum(0)
        s[0, D] += f.shape[0]
    return s


def apply_cmvn(x, stats):
    """ApplyCmvn with norm_vars: (x - mean) / sqrt(max(s1 / n - mean^2, 1e-20))."""
    D = stats.shape[1] - 1
    n = stats[0, D]
    mean = stats[0, :D] / n
    var = np.maximum(stats[1, :D] / n - mean ** 2, 1e-20)
    return (np.asarray(x, np.float64) - mean) / np.sqrt(var)


def batch(waves, o, draws=None, stats=None, T=None):
    """Time-major [T, B, D] features and mask [T, B] of a list of utterances (draws: per utterance [frames, W])."""
    feats = [features(w, o, None if draws is None else draws[b]) for b, w in enumerate(waves)]
    if stats is not None:
        feats = [apply_cmvn(f, stats) for f in feats]
    T = T or max(f.shape[0] for f in feats)
    out = np.zeros((T, len(waves), feats[0].shape[1]))
    mask = np.zeros((T, len(waves)))
    for b, f in enumerate(feats):
        out[:f.shape[0], b] = f
        mask[:f.shape[0], b] = 1
    return out, mask
