"""The filterbank oracle (tests/fbank_oracle.py) against torchaudio's independent restatement of Kaldi's
compute-fbank-feats, stored in tests/golden/fbank_kaldi_golden.npz by tests/golden/make_fbank_kaldi_golden.py.

The float64 records (every window, energy, power and DC option, pre-emphasis 0 / 0.5 / 1, band edges, 8 to 48 kHz,
10 to 126 bins, FFT sizes 8 to 512 with and without rounding, frame shifts of 1 sample to 201 ms, and DC, full-scale,
Nyquist, impulse and bin-centred signals) agree to 1e-9.  The float32 records hold silent and DC frames under both
raw_energy settings: every floored value is float32 log(FLT_EPSILON), exactly where the oracle floors, and the
others agree to float32 precision.  No GPU needed."""
import numpy as np
import pytest

import fbank_oracle as F
from fbank_helpers import LOG_EPS32, load_golden

RECORDS = load_golden()


def test_fixture_covers_every_option_and_signal():
    names = [r["name"] for r in RECORDS]
    assert len(names) == len(set(names))
    opts = [F.options(**r["options"]) for r in RECORDS]
    for key, values in dict(window_type=["povey", "hamming", "hanning", "rectangular"], use_power=[False],
                            remove_dc_offset=[False], raw_energy=[False], use_energy=[False],
                            round_to_power_of_two=[False], preemphasis_coefficient=[0.0, 0.5, 1.0],
                            sample_frequency=[8000.0, 11025.0, 16000.0, 22050.0, 44100.0, 48000.0]).items():
        assert set(values) <= {o[key] for o in opts}, key
    assert {F.frame_sizes(o)[2] for o in opts} >= {8, 16, 32, 64, 128, 256, 512}
    assert any(F.frame_sizes(o)[1] == 1 for o in opts) and any(F.frame_sizes(o)[1] > F.frame_sizes(o)[0] for o in opts)
    assert {r["signal"] for r in RECORDS} >= {"tones", "silence", "silent_middle", "dc", "full_scale", "nyquist",
                                              "bin_tones", "mel_tones", "impulses", "dc_noise"}
    assert all(r["wave"].dtype == np.int16 for r in RECORDS)
    assert any((r["wave"] == -32768).any() for r in RECORDS)


@pytest.mark.parametrize("rec", [r for r in RECORDS if r["dtype"] == "float64"], ids=lambda r: r["name"])
def test_oracle_matches_torchaudio_float64(rec):
    o = F.options(dither=0.0, **rec["options"])
    got = F.fbank(rec["wave"], o)
    want = rec["feats"]
    assert want.dtype == np.float64 and got.shape == want.shape
    assert np.abs(got - want).max() <= 1e-9, (rec["name"], np.abs(got - want).max())


@pytest.mark.parametrize("rec", [r for r in RECORDS if r["dtype"] == "float32"], ids=lambda r: r["name"])
def test_oracle_floors_as_torchaudio_float32(rec):
    o = F.options(dither=0.0, **rec["options"])
    got = F.fbank(rec["wave"], o)
    want = rec["feats"]
    assert want.dtype == np.float32 and got.shape == want.shape
    floored = want == LOG_EPS32
    assert floored.any()
    # the floor: float32 log(FLT_EPSILON), in the same places, for the raw and the windowed energy alike
    assert np.array_equal(got.astype(np.float32) == LOG_EPS32, floored), rec["name"]
    assert np.array_equal(got[floored].astype(np.float32), want[floored])
    if rec["signal"] in ("silence", "dc"):
        assert floored.all()
    else:
        assert np.abs(got - want)[~floored].max() <= 1e-4
