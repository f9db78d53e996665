"""Signals, the GPU-against-oracle comparison and the torchaudio fixture shared by the filterbank tests."""
import json
import os

import numpy as np
import pytest

import fbank_oracle as F
from helpers import ROOT, package

LIN_TOL = 5e-6
LOG_TOL = 5e-5
FEAT_TOL = 2e-3

GOLDEN = os.path.join(ROOT, "tests", "golden", "fbank_kaldi_golden.npz")
LOG_EPS32 = np.float32(np.log(np.float32(F.FLT_EPSILON)))     # a floored column, in float32


def torch_or_skip():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch


def signal(rng, n, fs=16000.0):
    """Three random tones over N(0, 300) noise, int16."""
    t = np.arange(n) / fs
    x = rng.normal(0, 300, size=n)
    for f in rng.uniform(100, 0.45 * fs, size=3):
        x += rng.uniform(500, 4000) * np.sin(2 * np.pi * f * t + rng.uniform(0, 6.3))
    return np.clip(np.round(x), -32768, 32767).astype(np.int16)


def waves(rng, lengths, fs=16000.0):
    return [signal(rng, n, fs) for n in lengths]


def int16(x):
    return np.clip(np.round(x), -32768, 32767).astype(np.int16)


def edge_signal(name, o, frames=6, seed=0):
    """An edge signal of `frames` frames under options o, int16."""
    W, S, P = F.frame_sizes(o)
    fs = o["sample_frequency"]
    n = W + (frames - 1) * S
    rng = np.random.RandomState(seed)
    t = np.arange(n) / fs
    if name == "tones":
        return signal(rng, n, fs)
    if name == "silence":
        return np.zeros(n, np.int16)
    if name == "silent_middle":                  # frames 2 .. frames-3 see nothing but zeros
        x = signal(rng, n, fs)
        x[2 * S:(frames - 3) * S + W] = 0
        return x
    if name == "dc":
        return np.full(n, 1234, np.int16)
    if name == "full_scale":                     # a 440 Hz square wave between -32768 and 32767
        return np.where(np.sin(2 * np.pi * 440 * t + 3.0) >= 0, 32767, -32768).astype(np.int16)
    if name == "nyquist":
        return np.where(np.arange(n) % 2 == 0, 32767, -32768).astype(np.int16)
    if name == "bin_tones":                      # exactly on FFT bins P/40, P/8 and 3P/8
        return int16(sum(8000 * np.cos(2 * np.pi * (k * P // 40) * np.arange(n) / P + 0.3 * k)
                         for k in (1, 5, 15)))
    if name == "mel_tones":                      # on the centres of the first, a middle and the last mel bin
        c = F.inverse_mel(F.mel_edges(o)[:, 1])
        return int16(sum(8000 * np.sin(2 * np.pi * f * t + 1.0) for f in (c[0], c[len(c) // 2], c[-1])))
    if name == "impulses":                       # at frame 0's samples 0 and W-1, and at frame 1's first (t = S)
        x = rng.normal(0, 3, size=n)
        for i, a in ((0, 30000), (W - 1, -30000), (S, 25000)):
            x[i] += a
        return int16(x)
    if name == "dc_noise":                       # a large DC offset under small noise
        return int16(20000 + rng.normal(0, 2, size=n))
    raise ValueError(name)


def make_fb(**kw):
    """(Fbank, oracle options) of oracle option overrides kw."""
    pkg = package()
    o = F.options(**kw)
    return pkg.Fbank(pkg.FbankOptions(**o)), o


def static_errors(got, want, lin, use_energy, errs):
    """The static columns got [n, D0] of one utterance against want [n, D0] (logs) and lin [n, bins] (the linear mel
    energies): linear relative to the frame's peak; logs absolutely where the energy is at least 1e-4 of the peak, and
    the log energy always."""
    ne = int(use_energy)
    peak = lin.max(1, keepdims=True)
    le = float((np.abs(np.exp(got[:, ne:]) - lin) / peak).max())
    strong = lin >= 1e-4 * peak
    ge = float(np.abs(got[:, ne:] - want[:, ne:])[strong].max())
    errs["lin"] = max(errs.get("lin", 0.0), le)
    errs["log"] = max(errs.get("log", 0.0), ge)
    if ne:
        errs["log"] = max(errs["log"], float(np.abs(got[:, 0] - want[:, 0]).max()))
    return errs


def check(feats, mask, wavs, o, draws=None, stats=None, errs=None):
    """The GPU's features [T, B, D] and mask against the oracle's; returns the worst errors."""
    feats, mask = feats.cpu().numpy().astype(np.float64), mask.cpu().numpy()
    T = feats.shape[0]
    want, wmask = F.batch(wavs, o, draws, stats, T=T)
    assert np.array_equal(mask, wmask)
    assert not feats[mask == 0].any(), "padded frames must be exactly 0"
    errs = {} if errs is None else errs
    e = float(np.abs(feats - want)[mask > 0].max())
    errs["feat"] = max(errs.get("feat", 0.0), e)
    assert e <= FEAT_TOL, ("features", e)
    if stats is None:
        for b, x in enumerate(wavs):
            st, lin = F.fbank(x, o, None if draws is None else draws[b], linear=True)
            static_errors(feats[:st.shape[0], b, :st.shape[1]], st, lin, o["use_energy"], errs)
        assert errs["lin"] <= LIN_TOL and errs["log"] <= LOG_TOL, errs
    return errs


def load_golden():
    """The torchaudio fixture: a list of records {name, options, signal, dtype, torchaudio, wave, feats}."""
    z = np.load(GOLDEN)
    recs = json.loads(str(z["records"]))
    for i, r in enumerate(recs):
        r["wave"] = z["wave%d" % i]
        r["feats"] = z["feats%d" % i]
    return recs
