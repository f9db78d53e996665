"""Generate tests/golden/fbank_kaldi_golden.npz: torchaudio's restatement of Kaldi's compute-fbank-feats
(torchaudio.compliance.kaldi.fbank), written independently of tests/fbank_oracle.py, at every option the front end
accepts and on edge signals, a few frames each.

Run from the repo root where torchaudio is installed:  python tests/golden/make_fbank_kaldi_golden.py
No test imports torchaudio: the fixture stores the int16 input waveforms and, per record, the options (the oracle's
names), the features [frames, D0] and the torchaudio version.

Records are computed in float64 with torch's default dtype float64, so the mel banks are not built in float32.
torchaudio floors the energies at float32's epsilon cast to the run's dtype; the float64 records are chosen so that
no floor binds (asserted below), which leaves the arithmetic to compare.  The floor cases (silent frames, DC with
remove_dc_offset, both raw_energy settings) are a separate float32 pass, where the floored values are float32
log(FLT_EPSILON).  Deltas and CMVN are not part of torchaudio's fbank.  The archive is written with fixed zip
timestamps, so a rerun reproduces it bit for bit.
"""
import io
import json
import os
import sys
import zipfile

import numpy as np
import torch
import torchaudio
import torchaudio.compliance.kaldi as kaldi

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import fbank_oracle as F  # noqa: E402
from fbank_helpers import GOLDEN, edge_signal  # noqa: E402


def ms(samples, fs=16000.0):
    """Milliseconds of `samples` at fs: exact in binary at 16 kHz."""
    return samples * 1000.0 / fs


# (name, oracle option overrides) on the tones signal, then (name, overrides, signal); dither is 0 throughout
TONES = [
    ("recipe", {}),
    ("hamming", dict(window_type="hamming")),
    ("hanning", dict(window_type="hanning")),
    ("rectangular", dict(window_type="rectangular")),
    ("magnitude", dict(use_power=False)),
    ("keep_dc", dict(remove_dc_offset=False)),
    ("preemph_0", dict(preemphasis_coefficient=0.0)),
    ("preemph_0.5", dict(preemphasis_coefficient=0.5)),
    ("preemph_1", dict(preemphasis_coefficient=1.0)),
    ("band_300_3400", dict(low_freq=300.0, high_freq=3400.0)),
    ("high_freq_-400", dict(high_freq=-400.0)),
    ("low_freq_0", dict(low_freq=0.0)),
    ("windowed_energy", dict(raw_energy=False)),
    ("energy_floor", dict(energy_floor=1.0)),
    ("no_energy", dict(use_energy=False)),
    ("bins_10", dict(num_mel_bins=10)),
    ("bins_126", dict(num_mel_bins=126)),
    ("8k_bins_95", dict(sample_frequency=8000.0, num_mel_bins=95)),
    ("8k", dict(sample_frequency=8000.0, num_mel_bins=23)),
    ("11025", dict(sample_frequency=11025.0)),
    ("22050_23ms", dict(sample_frequency=22050.0, frame_length=23.0)),
    ("44100_10ms", dict(sample_frequency=44100.0, frame_length=10.0)),
    ("48000_10ms", dict(sample_frequency=48000.0, frame_length=10.0)),
    ("shift_1", dict(frame_shift=ms(1))),
    ("shift_37ms", dict(frame_shift=37.0)),
    ("shift_201ms", dict(frame_shift=201.0)),
    ("W5_P8", dict(frame_length=ms(5), frame_shift=ms(3), low_freq=1000.0, num_mel_bins=4)),
    ("W8_P8", dict(frame_length=ms(8), frame_shift=ms(3), low_freq=1000.0, num_mel_bins=4, round_to_power_of_two=False)),
    ("W16_P16", dict(frame_length=ms(16), frame_shift=ms(7), num_mel_bins=4, round_to_power_of_two=False)),
    ("W32_P32", dict(frame_length=ms(32), frame_shift=ms(16), num_mel_bins=8, round_to_power_of_two=False)),
    ("W64_P64", dict(frame_length=ms(64), frame_shift=ms(32), num_mel_bins=10, round_to_power_of_two=False)),
    ("W100_P128", dict(frame_length=ms(100), frame_shift=ms(50), num_mel_bins=23)),
    ("W128_P128", dict(frame_length=ms(128), frame_shift=ms(50), num_mel_bins=23, round_to_power_of_two=False)),
    ("W256_P256", dict(frame_length=ms(256), frame_shift=ms(100), round_to_power_of_two=False)),
    ("W257_P512", dict(frame_length=ms(257), frame_shift=ms(100))),
    ("W511_P512", dict(frame_length=ms(511), frame_shift=ms(160))),
    ("W512_P512", dict(frame_length=ms(512), frame_shift=ms(160), round_to_power_of_two=False)),
]
EDGES64 = [
    ("dc_keep", dict(remove_dc_offset=False), "dc"),
    ("full_scale", {}, "full_scale"),
    ("nyquist", {}, "nyquist"),
    ("nyquist_rectangular", dict(window_type="rectangular"), "nyquist"),
    ("bin_tones", {}, "bin_tones"),
    ("bin_tones_8k", dict(sample_frequency=8000.0, num_mel_bins=23), "bin_tones"),
    ("mel_tones", {}, "mel_tones"),
    ("impulses", {}, "impulses"),
    ("impulses_rectangular", dict(window_type="rectangular"), "impulses"),
    ("impulses_hamming", dict(window_type="hamming"), "impulses"),
    ("dc_noise", {}, "dc_noise"),
]
EDGES32 = [
    ("silence", {}, "silence"),
    ("silence_windowed", dict(raw_energy=False), "silence"),
    ("silent_middle", {}, "silent_middle"),
    ("silent_middle_windowed", dict(raw_energy=False), "silent_middle"),
    ("dc", {}, "dc"),
    ("dc_windowed", dict(raw_energy=False), "dc"),
]
CASES = ([(n, kw, "tones", "float64") for n, kw in TONES] + [c + ("float64",) for c in EDGES64] +
         [c + ("float32",) for c in EDGES32])


def torchaudio_fbank(x, o, dtype):
    torch.set_default_dtype(dtype)
    try:
        wav = torch.as_tensor(np.asarray(x, np.float64), dtype=dtype)[None, :]
        out = kaldi.fbank(
            wav, dither=0.0, energy_floor=o["energy_floor"], frame_length=o["frame_length"],
            frame_shift=o["frame_shift"], high_freq=o["high_freq"], htk_compat=False, low_freq=o["low_freq"],
            num_mel_bins=o["num_mel_bins"], preemphasis_coefficient=o["preemphasis_coefficient"],
            raw_energy=o["raw_energy"], remove_dc_offset=o["remove_dc_offset"],
            round_to_power_of_two=o["round_to_power_of_two"], sample_frequency=o["sample_frequency"],
            snip_edges=True, use_energy=o["use_energy"], use_log_fbank=True, use_power=o["use_power"],
            window_type=o["window_type"])
    finally:
        torch.set_default_dtype(torch.float32)
    return out.numpy()


def main():
    torch.set_num_threads(1)
    arrays, records = {}, []
    for i, (name, kw, sig, dtype) in enumerate(CASES):
        o = F.options(dither=0.0, **kw)
        x = edge_signal(sig, o, frames=3 if name == "shift_201ms" else 6)
        feats = torchaudio_fbank(x, o, torch.float64 if dtype == "float64" else torch.float32)
        assert feats.shape == (F.num_frames(len(x), o), o["num_mel_bins"] + o["use_energy"]), (name, feats.shape)
        floor = np.log(np.array(F.FLT_EPSILON, feats.dtype))
        if dtype == "float64":
            assert (feats > floor).all(), (name, "a floor binds")
        else:
            assert (feats == floor).any(), (name, "no floor binds")
        arrays["wave%d" % i] = x
        arrays["feats%d" % i] = feats
        records.append(dict(name=name, options=kw, signal=sig, dtype=dtype, torchaudio=torchaudio.__version__))
    arrays["records"] = np.array(json.dumps(records))
    with zipfile.ZipFile(GOLDEN, "w", zipfile.ZIP_DEFLATED) as z:
        for key in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[key]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue(),
                       compress_type=zipfile.ZIP_DEFLATED)
    print("wrote %s: %d records, %d bytes" % (GOLDEN, len(records), os.path.getsize(GOLDEN)))


if __name__ == "__main__":
    main()
