"""Device memory of the model and front-end handles, through lvsr_device_bytes (the bytes every DeviceBuffer holds):
a destroyed handle gives back everything it allocated, whatever ran on it; each optional feature gives back what it
took when it is turned off; and a repeated call of the same shape allocates nothing (DESIGN.md section 3).

The counter is process-wide, so every measurement is a difference around this test's own handles, taken with the
garbage collector off: no other test's handle is released in the middle."""
import contextlib
import ctypes as C
import gc

import numpy as np
import pytest

from fbank_helpers import waves
from helpers import O, PYRAMID, make_recognizer, package
from oracle import lvsr_oracle_grad as G

pytestmark = pytest.mark.gpu

STAGES = ("create", "finalize", "encode", "cost_matrix", "alignment_stats", "beam_search", "train_step", "update")


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _lib():
    return package()._lib


def _bytes():
    return int(_lib().load().lvsr_device_bytes())


@contextlib.contextmanager
def _gc_off():
    gc.collect()
    gc.disable()
    try:
        yield
    finally:
        gc.enable()


def _destroy(rec):
    _lib().check(_lib().load().lvsr_model_destroy(rec._handle))
    rec._handle = None


def _setup(seed=3):
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=seed, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=4, T=60, seed=seed + 1)
    return cfg, params, (x, m, labels, lm)


def _algorithm(rec):
    pkg = package()
    tc = G.make_train_config(gradient_threshold=100.0, scale=0.01, momentum=0.5, epsilon=1e-6, max_norm=1.0)
    return pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(tc, dict(max_norm=1.0)))


def _batch(algo, batch):
    return dict(zip(algo.SOURCES, batch))


@pytest.mark.parametrize("stage", STAGES)
def test_destroy_returns_every_byte(stage):
    _torch()
    cfg, params, batch = _setup()
    x, m, labels, lm = batch
    with _gc_off():
        base = _bytes()
        rec = make_recognizer(cfg, params)
        rec._require_ready()
        assert _bytes() > base                     # the parameters and the status words
        upto = STAGES[:STAGES.index(stage) + 1]
        if "finalize" in upto:
            _lib().check(_lib().load().lvsr_model_finalize(rec._handle))
        if "encode" in upto:
            att, attm = rec.encode(x, m)
        if "cost_matrix" in upto:
            rec.cost_matrix(labels, lm, att, attm).cpu()
        if "alignment_stats" in upto:
            for B in (2, 4):                       # the second batch regrows the statistics' partial sums
                rec.validation_statistics(*(np.ascontiguousarray(a[:, :B]) for a in (x, m, labels, lm)))
        if "beam_search" in upto:
            rec.init_beam_search(4)
            rec.beam_search_many([{"recordings": x[:, 0]}], raise_on_failure=False)
        if "train_step" in upto:
            algo = _algorithm(rec)
            algo.cost_and_gradients(_batch(algo, batch))
        if "update" in upto:
            algo.process_batch(_batch(algo, batch))
            float(algo.last_cost.item())
        held = _bytes() - base
        _destroy(rec)
        assert _bytes() == base, (stage, held)


def _enable_disable(lib, h):
    """{feature: (enable, disable)} of every optional buffer group of a handle."""
    V = 32
    off = np.array([0, V], np.int64)                            # one state, a self loop for every label
    label = np.arange(1, V + 1, dtype=np.int32)
    nxt = np.zeros(V, np.int32)
    weight = np.linspace(0.5, 2.0, V).astype(np.float32)
    fusion = _lib().LvsrLmFusion(weight=0.5, am_beta=1.0, no_transition_cost=20.0)
    noise = _lib().LvsrAdaptiveNoise(init_sigma=1e-2, model_cost_coefficient=0.5, num_examples=40, seed=7)
    reg = _lib().LvsrRegularization(dropout=1, noise_level=0.05, penalty_coof=0.5, seed=11)
    clip = _lib().LvsrAdaptiveClipping(initial_threshold=10.0, decay_rate=0.9, burnin_period=3)
    return {
        "lm": (lambda: lib.lvsr_model_set_lm(h, 1, 0, off.ctypes.data, V, label.ctypes.data, nxt.ctypes.data,
                                             weight.ctypes.data, C.byref(fusion)),
               lambda: lib.lvsr_model_clear_lm(h)),
        "adaptive_noise": (lambda: lib.lvsr_train_set_adaptive_noise(h, C.byref(noise)),
                           lambda: lib.lvsr_train_set_adaptive_noise(h, None)),
        "regularization": (lambda: lib.lvsr_train_set_regularization(h, C.byref(reg)),
                           lambda: lib.lvsr_train_set_regularization(h, None)),
        "adaptive_clipping": (lambda: lib.lvsr_train_set_adaptive_clipping(h, C.byref(clip)),
                              lambda: lib.lvsr_train_set_adaptive_clipping(h, None)),
    }


def test_each_feature_gives_back_what_it_took():
    _torch()
    cfg, params, batch = _setup(seed=5)
    rec = make_recognizer(cfg, params)
    before = rec.cost(*batch)
    lib, h = _lib().load(), rec._require_ready()
    toggles = _enable_disable(lib, h)
    with _gc_off():
        taken = {}
        for cycle in range(3):
            for name, (enable, disable) in toggles.items():
                b0 = _bytes()
                _lib().check(enable())
                took = _bytes() - b0
                assert took > 0, name
                assert taken.setdefault(name, took) == took, (name, cycle, taken[name], took)
                _lib().check(disable())
                assert _bytes() == b0, (name, cycle)
        after = rec.cost(*batch)
        _destroy(rec)
    assert np.array_equal(after, before)


def test_steady_state_allocates_nothing():
    _torch()
    cfg, params, batch = _setup(seed=7)
    rec = make_recognizer(cfg, params)
    with _gc_off():
        held = []
        for _ in range(3):
            rec.cost(*batch)
            held.append(_bytes())
        assert held[1] == held[0] and held[2] == held[1], held
        algo = _algorithm(rec)
        held = []
        for _ in range(3):
            algo.process_batch(_batch(algo, batch))
            float(algo.last_cost.item())
            held.append(_bytes())
        assert held[1] == held[0] and held[2] == held[1], held
        _destroy(rec)


def test_frontend_destroy_returns_every_byte():
    torch = _torch()
    pkg = package()
    rng = np.random.RandomState(0)
    with _gc_off():
        base = _bytes()
        fb = pkg.Fbank(pkg.FbankOptions())
        held = [_bytes() - base]
        for B, n in ((1, 4000), (3, 8000), (6, 16000)):     # the frame and feature buffers grow with the batch
            fb.compute(waves(rng, [n] * B))
            torch.cuda.synchronize()
            held.append(_bytes() - base)
        assert held[0] > 0 and held[1] > held[0] and held[3] > held[1], held
        _lib().check(_lib().load().lvsr_frontend_destroy(fb._handle))
        fb._handle = None
        assert _bytes() == base
