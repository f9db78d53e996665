"""The filterbank oracle (tests/fbank_oracle.py) pinned by answers derivable by hand, the option refusals of
lvsr_frontend_create and the ctypes mirror of lvsr_fbank_options.  No GPU needed."""
import ctypes
import os
import re

import numpy as np
import pytest

import fbank_oracle as F
from helpers import ROOT, package

O16 = F.options(dither=0.0)


@pytest.mark.parametrize("N,frames", [(399, 0), (400, 1), (559, 1), (560, 2)])
def test_frame_count(N, frames):
    assert F.frame_sizes(O16) == (400, 160, 512)
    assert F.num_frames(N, O16) == frames


def test_window_values():
    W = 400
    povey, hamming = F.window(F.options(window_type="povey")), F.window(F.options(window_type="hamming"))
    assert povey[0] == 0 and abs(povey[W - 1]) < 1e-12
    assert hamming[0] == pytest.approx(0.08) and hamming[W - 1] == pytest.approx(0.08)
    # (W - 1) / 2 = 199.5 falls between samples: the formulas there give the peak, 1
    a = 2 * np.pi * 199.5 / (W - 1)
    assert (0.5 - 0.5 * np.cos(a)) ** 0.85 == pytest.approx(1.0) and 0.54 - 0.46 * np.cos(a) == pytest.approx(1.0)
    assert povey[199] == pytest.approx(povey[200]) and povey[199] > 0.9999
    assert np.all(povey <= 1) and np.all(hamming <= 1)


def test_mel_filter_edges_in_hz():
    # mel(20) = 1127 ln(1 + 20/700) = 31.7486, mel(8000) = 1127 ln(1 + 8000/700) = 2840.0377, step = 68.4947 over 41
    # steps; bin 0: 20 Hz | 700 (e^{100.2433/1127} - 1) = 65.116 Hz | 113.059 Hz; bin 39: 7004.24 | 7486.99 | 8000 Hz
    hz = F.inverse_mel(F.mel_edges(O16))
    assert hz.shape == (40, 3)
    np.testing.assert_allclose(hz[0], [20.0, 65.116, 113.059], atol=2e-3)
    np.testing.assert_allclose(hz[39], [7004.237, 7486.994, 8000.0], atol=2e-3)
    np.testing.assert_allclose(hz[1:, 0], hz[:-1, 1])             # each bin starts at its left neighbour's centre


def test_every_filter_peaks_at_its_centre_and_never_weights_nyquist():
    banks = F.mel_banks(O16)
    assert banks.shape == (40, 257)
    assert not banks[:, 256].any()
    edges = F.mel_edges(O16)
    np.testing.assert_allclose(F.triangle(edges[:, 1], edges).diagonal(), 1.0)
    fft_mel = F.mel(np.arange(256) * 16000.0 / 512)
    for b in range(40):
        assert banks[b].max() <= 1.0
        assert np.argmax(banks[b]) == np.argmin(np.abs(fft_mel - edges[b, 1])), b
        nz = np.flatnonzero(banks[b])
        assert np.all(np.diff(nz) == 1) and (fft_mel[nz] > edges[b, 0]).all() and (fft_mel[nz] < edges[b, 2]).all()


def test_parseval():
    rng = np.random.RandomState(0)
    x = rng.randint(-3000, 3000, size=16000).astype(np.float64)
    win, spec, _ = F.process_frames(x, O16)
    full = spec[:, 0] + spec[:, -1] + 2 * spec[:, 1:-1].sum(1)
    np.testing.assert_allclose(full, 512 * (win ** 2).sum(1), rtol=1e-10)


def test_pure_tone_lands_in_the_nearest_bin():
    t = np.arange(8000) / 16000.0
    x = np.round(8000 * np.sin(2 * np.pi * 1000 * t))
    _, energies = F.fbank(x, O16, linear=True)
    centres = F.inverse_mel(F.mel_edges(O16)[:, 1])
    assert (np.argmax(energies, axis=1) == np.argmin(np.abs(centres - 1000))).all()


def test_constant_signal_floors_energy_and_bins():
    f = F.fbank(np.full(4000, 1234.0), O16)
    np.testing.assert_array_equal(f, np.log(F.FLT_EPSILON))
    assert f.shape == (23, 41)               # 1 + (4000 - 400) // 160 frames


def test_delta_of_ramp_and_delta_delta_of_square():
    T = 12
    t = np.arange(T, dtype=np.float64)[:, None]
    d = F.add_deltas(t, order=1, window=2)[:, 1]
    np.testing.assert_allclose(d[2:T - 2], 1.0)
    # clamped: t = 0 sees [0, 0, 0, 1, 2] -> 0.5, t = 1 sees [0, 0, 1, 2, 3] -> 0.8, and mirrored at the end
    np.testing.assert_allclose(d[[0, 1, T - 2, T - 1]], [0.5, 0.8, 0.8, 0.5])
    dd = F.add_deltas(t ** 2, order=2, window=2)[:, 2]
    np.testing.assert_allclose(dd[4:T - 4], 2.0)
    np.testing.assert_allclose(F.delta_scales(2, 2)[2] * 100, [4, 4, 1, -4, -10, -4, 1, 4, 4])


def test_cmvn_of_a_ragged_set_normalises_it():
    rng = np.random.RandomState(1)
    feats = [rng.normal(3.0, 2.0, size=(n, 5)) * np.arange(1, 6) for n in (7, 30, 1, 64)]
    s = F.cmvn_stats(feats)
    assert s.shape == (2, 6) and s[0, 5] == 102 and s[1, 5] == 0
    allf = np.concatenate([F.apply_cmvn(f, s) for f in feats])
    np.testing.assert_allclose(allf.mean(0), 0.0, atol=1e-12)
    np.testing.assert_allclose(allf.var(0), 1.0, rtol=1e-12)


def _create(**kw):
    pkg = package()
    lib = pkg._lib.load()
    h = ctypes.c_void_p()
    s = pkg.FbankOptions(**kw)._struct()
    rc = lib.lvsr_frontend_create(ctypes.byref(s), ctypes.byref(h))
    msg = (lib.lvsr_last_error() or b"").decode("utf-8", "replace")
    if rc == 0:
        lib.lvsr_frontend_destroy(h)
    return rc, msg


@pytest.mark.parametrize("kw,message", [
    (dict(snip_edges=False), "snip_edges false is not supported"),
    (dict(vtln_warp=0.9), "VTLN warping is not supported"),
    (dict(htk_compat=True), "htk_compat true is not supported"),
    (dict(use_log_fbank=False), "use_log_fbank false is not supported"),
    (dict(frame_length=40.0), "frame_length 40 ms is 640 samples: longer than the 512-point FFT supports"),
    (dict(round_to_power_of_two=False), "round_to_power_of_two false needs a frame of a power-of-two length"),
    (dict(num_mel_bins=200), "num_mel_bins 200 too large"),
    (dict(high_freq=9000.0), "bad mel band edges"),
    (dict(delta_order=4), "delta_order 4 not in [0, 3]"),
])
def test_options_are_refused(kw, message):
    rc, msg = _create(**kw)
    assert rc != 0 and message in msg, msg


def test_recipe_options_pass_the_checks():
    rc, msg = _create()                      # past the checks: fails on the device only where there is none
    assert rc == 0 or "no CUDA device" in msg or "cuda" in msg.lower(), msg
    with pytest.raises(TypeError, match="unknown fbank options: num_ceps"):
        package().FbankOptions(num_ceps=13)
    with pytest.raises(ValueError, match="window_type 'blackman' unsupported"):
        package().FbankOptions(window_type="blackman")._struct()


def test_header_struct_matches_ctypes_mirror():
    with open(os.path.join(ROOT, "include", "lvsr_b200.h")) as fh:
        src = fh.read()
    body = re.search(r"typedef struct \{([^}]*)\} lvsr_fbank_options;", src).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"(double|uint64_t|int32_t)\s+(\w+);", body)
    ctypes_of = {"double": ctypes.c_double, "uint64_t": ctypes.c_uint64, "int32_t": ctypes.c_int32}
    mirror = package()._lib.LvsrFbankOptions._fields_
    assert [(n, ctypes_of[t]) for t, n in fields] == list(mirror)
    assert ctypes.sizeof(package()._lib.LvsrFbankOptions) == 9 * 8 + 8 + 12 * 4
    for name in ("lvsr_frontend_create", "lvsr_frontend_destroy", "lvsr_frontend_num_frames", "lvsr_frontend_feature_dim",
                 "lvsr_frontend_compute", "lvsr_frontend_accumulate_cmvn", "lvsr_frontend_apply_cmvn",
                 "lvsr_frontend_dither_sample"):
        assert name in package()._lib.SIGNATURES and re.search(r"\b%s\(" % name, src), name
