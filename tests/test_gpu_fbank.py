"""The filterbank front end (csrc/fbank.cu, frontend.py) against the float64 oracle of tests/fbank_oracle.py.

Kaldi's arithmetic is float32 too, so a weak mel bin carries FFT round-off relative to its frame's strongest one.
The comparisons, on signals of tones over noise in int16 units:
  * static columns (log energy and log mel bins, before deltas and CMVN): exp of the GPU's log mel bins against the
    oracle's linear mel energies, relative to the frame's largest (LIN_TOL); the logs themselves, absolutely, where
    the energy is at least 1e-4 of that largest (LOG_TOL);
  * every feature column after deltas and CMVN, absolutely (FEAT_TOL): weak bins included, so this is the loosest;
  * frames past an utterance's end: exactly 0, mask 0.
Measured worsts over this file on an H100 80GB HBM3 (700 W): linear 1.4e-6, log 8.4e-6, features 7.1e-4 (80 bins,
whose narrowest low bins are the weakest after pre-emphasis; 2.1e-4 at the recipe's 40).
"""
import os
import subprocess
import sys
import wave

import numpy as np
import pytest

import fbank_oracle as F
from compat_helpers import BASE_YAML, COMPAT
import fbank_helpers as H
from helpers import ROOT, O, make_recognizer, package

pytestmark = pytest.mark.gpu

CONFIGS = [
    dict(),
    dict(sample_frequency=8000.0, num_mel_bins=23),
    dict(sample_frequency=8000.0, num_mel_bins=40, window_type="hamming"),
    dict(num_mel_bins=80),
    dict(num_mel_bins=40, use_energy=False, delta_order=0),
    dict(raw_energy=False),
    dict(energy_floor=1.0),
    dict(window_type="hamming", raw_energy=False, num_mel_bins=23),
    dict(sample_frequency=8000.0, use_energy=False, energy_floor=1.0),
    dict(num_mel_bins=23, delta_order=0, energy_floor=1.0),
]


@pytest.mark.parametrize("cmvn", [False, True], ids=["raw", "cmvn"])
@pytest.mark.parametrize("kw", CONFIGS, ids=lambda kw: "-".join("%s=%s" % i for i in kw.items()) or "recipe")
def test_features_match_oracle(kw, cmvn):
    H.torch_or_skip()
    fb, o = H.make_fb(dither=0.0, **kw)
    W, S, _ = F.frame_sizes(o)
    rng = np.random.RandomState(len(kw) * 7 + int(cmvn))
    lengths = [W, W + S - 1, W + 5 * S, W + 5 * S + 1, W + 17 * S - 1, 3 * W + 11, int(o["sample_frequency"])]
    waves = H.waves(rng, lengths, o["sample_frequency"])
    assert fb.feature_dim == (o["num_mel_bins"] + o["use_energy"]) * (o["delta_order"] + 1)
    assert [fb.num_frames(n) for n in lengths] == [F.num_frames(n, o) for n in lengths]
    stats = None
    if cmvn:
        stats = F.cmvn_stats([F.features(x, o) for x in waves])
    feats, mask = fb.compute(waves, cmvn=stats)
    print(kw, cmvn, H.check(feats, mask, waves, o, stats=stats))


@pytest.mark.parametrize("B", [1, 7, 64, 129])
def test_batches(B):
    H.torch_or_skip()
    fb, o = H.make_fb(dither=0.0)
    rng = np.random.RandomState(B)
    if B == 1:
        lengths = [400 + 1999 * 160]                        # 20 s: 2000 frames
    else:
        edges = [400, 399 + 160, 400 + 160, 401 + 160, 400 + 7 * 160 - 1, 400 + 7 * 160 + 1]
        lengths = (edges + list(rng.randint(400, 16000 * (3 if B < 100 else 1), size=B)))[:B]
    waves = H.waves(rng, lengths)
    feats, mask = fb.compute(waves, T=max(fb.num_frames(n) for n in lengths) + 3)
    assert feats.shape[0] == max(F.num_frames(n, o) for n in lengths) + 3
    print(B, H.check(feats, mask, waves, o))


def test_tensor_input_and_short_utterance_refused():
    torch = H.torch_or_skip()
    fb, o = H.make_fb(dither=0.0, delta_order=0)
    rng = np.random.RandomState(3)
    waves = H.waves(rng, [4000, 2500, 3333])
    x = torch.zeros((3, 4001), dtype=torch.float32, device="cuda")        # row stride padded to 4004 inside
    for b, w in enumerate(waves):
        x[b, :len(w)] = torch.as_tensor(w.astype(np.float32))
    got, m = fb.compute(x, lengths=[len(w) for w in waves])
    want, wm = fb.compute(waves)
    assert torch.equal(got, want) and torch.equal(m, wm)
    with pytest.raises(RuntimeError, match="utterance 1 is shorter than one frame"):
        fb.compute([waves[0], waves[1][:399]])


def test_dither_is_replayable_and_keyed_by_seed():
    torch = H.torch_or_skip()
    fb, o = H.make_fb(dither=1.0, seed=7)
    rng = np.random.RandomState(9)
    waves = H.waves(rng, [5000, 400, 3210])
    a, m = fb.compute(waves)
    b, _ = fb.compute(waves)
    assert torch.equal(a, b)
    draws = fb.dither_sample(len(waves), a.shape[0]).cpu().numpy()
    assert abs(draws.mean()) < 0.05 and abs(draws.std() - 1) < 0.05
    print(H.check(a, m, waves, o, draws=list(draws)))
    other, _ = H.make_fb(dither=1.0, seed=8)
    c, _ = other.compute(waves)
    assert not torch.equal(a, c)
    quiet, _ = H.make_fb(dither=0.0)
    d1, _ = quiet.compute(waves)
    d2, _ = quiet.compute(waves)
    assert torch.equal(d1, d2)


def test_cmvn_accumulation_and_application():
    torch = H.torch_or_skip()
    pkg = package()
    fb, o = H.make_fb(dither=0.0)
    rng = np.random.RandomState(11)
    waves = H.waves(rng, [8000, 400, 5000, 12345, 999])
    feats, mask = fb.compute(waves)
    cmvn = pkg.GlobalCmvn(fb)
    cmvn.accumulate(feats, mask)
    got = cmvn.stats
    f64, m = feats.cpu().numpy().astype(np.float64), mask.cpu().numpy()
    want = F.cmvn_stats([f64[:int(m[:, b].sum()), b] for b in range(len(waves))])
    assert np.abs(got - want).max() <= 1e-9 * np.abs(want).max()
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-9 * np.abs(want).max())
    # two batches give the one batch's stats
    two = pkg.GlobalCmvn(fb)
    for part in (waves[:2], waves[2:]):
        x, mm = fb.compute(part)
        two.accumulate(x, mm)
    np.testing.assert_allclose(two.stats, got, rtol=1e-12)
    # apply in place == compute with the stats == the oracle's ApplyCmvn of the GPU features
    normed = cmvn.apply(feats.clone(), mask)
    direct, _ = fb.compute(waves, cmvn=cmvn)
    assert torch.equal(normed, direct)
    ref = np.where(m[..., None] > 0, F.apply_cmvn(f64, got), 0.0)
    assert np.abs(direct.cpu().numpy() - ref).max() < 1e-5
    # stats written and read as numpy
    path = os.path.join(os.environ.get("TMPDIR", "/tmp"), "fbank_cmvn_%d.npy" % os.getpid())
    cmvn.save(path)
    assert np.array_equal(pkg.GlobalCmvn.load(fb, path).stats, got)
    os.remove(path)


def test_compute_on_a_non_blocking_stream():
    torch = H.torch_or_skip()
    fb, o = H.make_fb(dither=1.0, seed=3)
    rng = np.random.RandomState(12)
    waves = H.waves(rng, [16000, 7000, 401])
    want, wm = fb.compute(waves)
    cmvn = package().GlobalCmvn(fb)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got, gm = fb.compute(waves)
        cmvn.accumulate(got, gm)
        normed, _ = fb.compute(waves, cmvn=cmvn)
    s.synchronize()
    assert torch.equal(got, want) and torch.equal(gm, wm)
    back, _ = fb.compute(waves, cmvn=cmvn)                      # back on the default stream: ordered after s
    assert torch.equal(back, normed)


def test_end_to_end_recognizer_on_gpu_features():
    """The CUDA features go straight into a 123-feature recognizer (wsj_jan_new-shaped, small)."""
    H.torch_or_skip()
    fb, o = H.make_fb(dither=0.0)
    rng = np.random.RandomState(21)
    waves = H.waves(rng, [16000, 9000, 12000])
    raw, _ = fb.compute(waves)
    stats = F.cmvn_stats([F.features(x, o) for x in waves])
    feats, mask = fb.compute(waves, cmvn=stats)
    want, wmask = F.batch(waves, o, stats=stats)
    cfg = O.make_config(num_features=123, dims_bidir=[128, 128], subsample=[1, 2], dim_dec=128, conv_n=8,
                        conv_num_filters=10, num_phonemes=32, post_merge_dims=[128], maxout_pieces=2,
                        max_decoded_length_scale=3.0)
    params = O.init_params(cfg, seed=5, scale=10.0)
    rec = make_recognizer(cfg, params)
    att, attm = rec.encode(feats, mask)                          # device tensors in, no copy through the host
    assert att.shape[0] == rec.encoded_length(feats.shape[0])
    L = 12
    labels = rng.randint(0, cfg["num_phonemes"] - 1, size=(L, 3)).astype(np.int64)
    lm = np.ones((L, 3), np.float32)
    got = rec.cost(feats.cpu().numpy(), mask.cpu().numpy(), labels, lm)
    ref = O.recognizer_cost(cfg, params, want, wmask, labels, lm)
    assert np.abs(got - ref).max() <= 1e-4 * np.abs(ref).max(), (got, ref)
    f = feats.cpu().numpy()
    n = [int(v) for v in mask.cpu().numpy().sum(0)]
    rec.init_beam_search(3)
    many = rec.beam_search_many([{"recordings": f[:n[b], b]} for b in range(3)], raise_on_failure=False)
    for b in range(3):
        try:
            w = O.beam_search(cfg, params, want[:n[b], b], 3)
        except O.CandidateNotFoundError:
            assert many[b] is None
            continue
        assert many[b] is not None and many[b][0] == w[0]


def _write_wav(path, x, fs=16000):
    with wave.open(path, "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(fs)
        w.writeframes(x.astype("<i2").tobytes())


def test_featurize_writes_the_oracle_features_and_compat_searches_them(tmp_path, capsys):
    H.torch_or_skip()
    rng = np.random.RandomState(31)
    texts = {"train": ["abc", "bad", "cab", "dab", "a", "ccd"], "valid": ["ab", "dc"]}
    waves = {}
    for part, ts in texts.items():
        lines, waves[part] = [], []
        for i, t in enumerate(ts):
            x = H.signal(rng, int(rng.randint(4000, 9000)))
            waves[part].append(x)
            _write_wav(str(tmp_path / ("%s%d.wav" % (part, i))), x)
            lines.append("%s_%d %s%d.wav %s" % (part, i, part, i, t))
        (tmp_path / ("%s.lst" % part)).write_text("\n".join(lines) + "\n")
    npz = str(tmp_path / "data.npz")
    subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "featurize.py"), "--part",
                           "train=" + str(tmp_path / "train.lst"), "--part", "valid=" + str(tmp_path / "valid.lst"),
                           "--out", npz, "--dither", "0"])
    z = np.load(npz)
    o = F.options(dither=0.0)
    stats = F.cmvn_stats([F.features(x, o) for x in waves["train"]])
    assert z["characters"].tolist() == ["a", "b", "c", "d", "</s>"] and int(z["num_labels"]) == 5
    assert (np.abs(z["cmvn"] - stats).max(1) <= 1e-6 * np.abs(stats).max(1)).all()
    for part in texts:
        want = np.concatenate([F.apply_cmvn(F.features(x, o), stats) for x in waves[part]])
        assert z[part + "_features"].shape == want.shape == (len(want), 123)
        assert np.abs(z[part + "_features"] - want).max() <= H.FEAT_TOL
        assert z[part + "_labels"].tolist() == ["abcd".index(c) for t in texts[part] for c in t]
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as LC
    import lvsr.main as M
    base = str(tmp_path / "base.yaml")
    with open(base, "w") as f:
        f.write(BASE_YAML.format(npz=npz))
    cfg = LC.Configuration(base, "$LVSR/lvsr/configs/schema.yaml", [])
    out = str(tmp_path / "model.tar")
    M.train(cfg, out)
    capsys.readouterr()
    single = LC.Configuration(base, "$LVSR/lvsr/configs/schema.yaml", [("monitoring.search.beam_size", "2")])
    M.search(single, None, out, "valid", None, None, str(tmp_path / "decoded.txt"), False, 1)
    assert "Average CER:" in capsys.readouterr().out
