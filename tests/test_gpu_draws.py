"""The training step's random draws on the GPU against their numpy restatement (tests/draws_oracle.py), which derives
them from Philox-4x32-10 and Box-Muller alone rather than replaying the library's kernels:

  * dropout multipliers bit for bit: at bench.py's 1500 x 64 x 40 batch (3.84 M elements, several passes of the
    kernel's grid-stride loop), at feature counts that are not a multiple of 32 or exceed 128, one utterance, shard
    offsets r * 64, updates 0, 1 and 2^31 + 5, and a seed whose high word is set;
  * weight-noise and adaptive-noise eps to draws_oracle.eps_bar (a few float32 ulps of max(r, 1), from the CUDA math
    functions' error bounds; the library builds without fast math), exact zeros on the padding between parameters
    and on the parameters weight noise leaves alone, a parameter whose element count is not a multiple of 4, on
    bench.py's model and on a TIMIT-sized one, at updates whose high word is set too."""
import ctypes as C

import numpy as np
import pytest

import bench
import content_oracle as CO
import draws_oracle as D
import regularization_oracle as RO
from helpers import O, bench_recognizer, make_recognizer, package

pytestmark = pytest.mark.gpu

HIGH_SEED = 0x9E3779B97F4A7C15
TIMIT = dict(num_features=123, dims_bidir=[128, 128], subsample=[1, 2], dim_dec=128, dim_matcher=128,
             num_phonemes=63, post_merge_dims=[128], maxout_pieces=2)
UPDATES = [0, 1, (1 << 31) + 5, (1 << 32) + 3]


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _bench_recognizer():
    rec = bench_recognizer()
    rec.initialize(seed=3)
    return rec


def _set_regularization(rec, **kw):
    pkg = package()
    cfg = pkg._lib.LvsrRegularization(**kw)
    pkg._lib.check(pkg._lib.load().lvsr_train_set_regularization(rec._require_ready(), C.byref(cfg)))


def _mask(rec, update, offset, T, B, F):
    torch = _torch()
    buf = torch.full((T, B, F), 7.0, dtype=torch.float32, device=rec.device)
    pkg = package()
    pkg._lib.check(pkg._lib.load().lvsr_train_dropout_mask(rec._require_ready(), update, offset, T, B, F,
                                                           buf.data_ptr(), rec._stream()))
    return buf.cpu().numpy()


def _mask_cases():
    W = bench.TRAIN_WORKLOAD
    return [
        ("bench", 3, 0, 0, (W["T"], W["B"], W["F"])),
        ("bench_update1", 3, 1, 0, (W["T"], W["B"], W["F"])),
        ("F123", 3, 1, 0, (50, 8, 123)),
        ("F1000", 3, 0, 0, (20, 8, 1000)),
        ("B1", 3, 0, 0, (300, 1, 40)),
        ("update_2^31+5", 3, (1 << 31) + 5, 0, (100, 16, 40)),
        ("high_seed", HIGH_SEED, 2, 0, (100, 16, 40)),
    ] + [("shard%d" % r, 3, 0, r * 64, (200, 64, 40)) for r in range(8)]


@pytest.mark.parametrize("name,seed,update,offset,shape", _mask_cases(), ids=[c[0] for c in _mask_cases()])
def test_dropout_mask_is_the_philox_bit_of_each_element(name, seed, update, offset, shape):
    _torch()
    rec = make_recognizer(O.make_config(**dict(TIMIT, num_features=40)), None)
    rec.initialize(seed=1)
    _set_regularization(rec, dropout=1, noise_level=0.0, penalty_coof=0.0, seed=seed)
    got = _mask(rec, update, offset, *shape)
    want = D.dropout_multiplier(seed, update, offset, *shape)
    bad = np.argwhere(got != want)
    assert bad.size == 0, (bad.shape[0], [tuple(int(i) for i in b) for b in bad[:5]])


def _spans(algo, rec):
    """(flat spans in parameter order, flat length, names); the spans are draws_oracle.flat_layout's."""
    off = algo._offsets()
    spans = list(off.values())
    counts = [int(np.prod(s)) for s in rec.parameter_shapes().values()]
    assert list(off) == list(rec.parameter_shapes())
    assert (spans, algo._n) == D.flat_layout(counts)
    return spans, algo._n, list(off)


def _check_eps(got, want, rad, spans, n):
    inside = np.zeros(n, bool)
    for o, c in spans:
        inside[o:o + c] = True
    assert not got[~inside].any()
    err = np.abs(got.astype(np.float64) - want)
    ratio = err / D.eps_bar(rad)
    assert ratio.max() <= 1.0, (int(ratio.argmax()), float(err.max()))
    return float(ratio.max())


def _flat_weight_noise_eps(rec, n, update):
    torch = _torch()
    pkg = package()
    buf = torch.full((n,), 7.0, dtype=torch.float32, device=rec.device)
    pkg._lib.check(pkg._lib.load().lvsr_train_weight_noise_sample(rec._require_ready(), update, buf.data_ptr(),
                                                                  rec._stream()))
    return buf.cpu().numpy()


@pytest.mark.parametrize("model", ["bench", "timit_content"])
@pytest.mark.parametrize("seed", [5, HIGH_SEED], ids=["seed5", "high_seed"])
def test_weight_noise_eps_matches_philox_box_muller(model, seed):
    _torch()
    pkg = package()
    if model == "bench":
        rec = _bench_recognizer()
    else:
        rec = make_recognizer(CO.make_config(**TIMIT), None)
        rec.initialize(seed=1)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]),
                               regularization=dict(noise=0.05, seed=5))
    algo.initialize()
    _set_regularization(rec, dropout=0, noise_level=0.05, penalty_coof=0.0, seed=seed)
    spans, n, names = _spans(algo, rec)
    subject = [RO.is_noise_subject(k) for k in names]
    assert not all(subject) and any(subject)
    if model != "bench":
        assert any(s and c % 4 for s, (o, c) in zip(subject, spans)), "no subject whose count is not a multiple of 4"
    worst = 0.0
    for update in UPDATES:
        got = _flat_weight_noise_eps(rec, n, update)
        want, rad = D.weight_noise_eps(seed, update, spans, n, subject)
        for (o, c), s, k in zip(spans, subject, names):
            if not s:
                assert not got[o:o + c].any(), k
        worst = max(worst, _check_eps(got, want, rad, spans, n))
    print("%s seed %#x: worst weight-noise eps error / bar %.3f over %d elements" % (model, seed, worst, n))


@pytest.mark.parametrize("seed", [7, HIGH_SEED], ids=["seed7", "high_seed"])
def test_adaptive_noise_eps_matches_philox_box_muller(seed):
    torch = _torch()
    pkg = package()
    rec = make_recognizer(O.make_config(**TIMIT), None)
    rec.initialize(seed=1)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]),
                               adaptive_noise=dict(num_examples=40, init_sigma=1e-2, seed=seed))
    algo.initialize()
    spans, n, _ = _spans(algo, rec)
    assert any(c % 4 for o, c in spans)
    lib, h = pkg._lib.load(), rec._require_ready()
    worst = 0.0
    for update in UPDATES:
        buf = torch.full((n,), 7.0, dtype=torch.float32, device=rec.device)
        pkg._lib.check(lib.lvsr_train_noise_sample(h, update, buf.data_ptr(), rec._stream()))
        want, rad = D.adaptive_noise_eps(seed, update, spans, n)
        worst = max(worst, _check_eps(buf.cpu().numpy(), want, rad, spans, n))
    print("adaptive noise seed %#x: worst eps error / bar %.3f over %d elements" % (seed, worst, n))
