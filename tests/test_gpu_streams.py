"""The C ABI's stream contract on a non-blocking stream (include/lvsr_b200.h): every entry point that takes a stream
runs in that stream's order, and every host call without one (parameters, gradient norm, optimizer reset, noise
parameters) takes effect after all work queued on the handle.

Every case runs twice: on the legacy default stream, which orders everything after everything else, and on a
torch.cuda.Stream(), which the driver must report as CU_STREAM_NON_BLOCKING (else the arm proves nothing and fails).
Before each call under test a spin of SPIN clock cycles is queued on the stream, so when the host gets control back
the library's work is still queued behind it: a read or write that is not ordered after that work sees stale data
every time, not by chance.  That holds only once the handle is warm: the first call at a shape sizes the workspace
(Arena::reserve synchronises the stream) and the first call after the parameters changed re-packs the weights (which
synchronises too), so each handle under test first makes the same calls at the same shapes without a spin.  No host
synchronisation (.item(), .cpu()) stands between a call and the host read under test.  The answers must be
bit-identical to a serial run on the default stream and within the oracle's bounds."""
import ctypes
from collections import OrderedDict

import numpy as np
import pytest

import adaptive_noise_oracle as AN
from helpers import O, PYRAMID, make_recognizer, package, rel_err
from oracle import lvsr_oracle_grad as G
from test_gpu_lm import LO_DEFAULTS, _peaky, _recognizer, lm_file  # noqa: F401  (lm_file: the module's LM fixture)

pytestmark = pytest.mark.gpu

TOL = 1e-4
SPIN = 200_000_000                  # cycles of torch.cuda._sleep: about 0.1 s on an H100
CU_STREAM_NON_BLOCKING = 1
ATT = "/recognizer/generator/att_trans/conv_att"
BIAS = ATT + "/energy_comp/linear.b"
ENERGY_BIAS = dict(logistic=-0.5, relu=1.0)


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _side_stream():
    """A pool stream, checked through the driver to be non-blocking: the legacy stream does not wait for it."""
    torch = _torch()
    s = torch.cuda.Stream()
    flags = ctypes.c_uint(0)
    cuda = ctypes.CDLL("libcuda.so.1")
    assert cuda.cuStreamGetFlags(ctypes.c_void_p(s.cuda_stream), ctypes.byref(flags)) == 0
    assert flags.value & CU_STREAM_NON_BLOCKING, "torch.cuda.Stream() is not CU_STREAM_NON_BLOCKING: the test is void"
    return s


@pytest.fixture(params=["default", "side"])
def stream(request):
    torch = _torch()
    if request.param == "default":
        s = torch.cuda.default_stream()
        assert s.cuda_stream == 0          # the legacy stream
        return s
    return _side_stream()


def _delay(s):
    """Queue SPIN cycles on s: whatever is enqueued next on s is still pending when the host returns."""
    torch = _torch()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SPIN)
    assert not s.query()


def _on(s, fn, *args, delay=True, **kw):
    """fn(*args) with s current, behind a queued spin."""
    torch = _torch()
    with torch.cuda.stream(s):
        if delay:
            _delay(s)
        return fn(*args, **kw)


def _dev(s, *arrays):
    """Device copies made on the default stream and ordered before s: the caller orders its own data."""
    torch = _torch()
    out = [None if a is None else torch.as_tensor(np.ascontiguousarray(a), device="cuda") for a in arrays]
    s.wait_stream(torch.cuda.default_stream())
    return out


def _np(t):
    return {k: v.cpu().numpy() for k, v in t.items()} if isinstance(t, dict) else t.cpu().numpy()


def _equal(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_equal(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))
    return np.array_equal(np.asarray(a), np.asarray(b))


# ---- inference ---------------------------------------------------------------------------------------------------

def _inference(rec, s, x, m, labels, lm, delay):
    """encode, preprocess, cost_matrix(return_all), the host cost and greedy generate, on s."""
    xd, md, yd, ymd = _dev(s, x, m, labels, lm)
    att, attm = _on(s, rec.encode, xd, md, delay=delay)
    P = _on(s, rec.preprocess, att, delay=delay)
    out = _on(s, rec.cost_matrix, yd, ymd, att, attm, return_all=True, delay=delay)
    cost = _on(s, rec.cost, x, m, labels, lm, delay=delay)
    gen = _on(s, rec.generate, x, m, n_steps=8, sample=False, delay=delay)
    s.synchronize()
    return dict(att=att.cpu().numpy(), attm=attm.cpu().numpy(), P=P.cpu().numpy(), all=_np(out), cost=cost,
                gen=gen)


@pytest.mark.parametrize("decoder", ["persistent", "stepwise"])
def test_inference_is_ordered_on_the_stream(stream, decoder, monkeypatch):
    """Every inference entry point behind a queued spin: the persistent decoder and the step-wise kernels
    (LVSR_NO_DEC_SCAN) give the serial default-stream answers bit for bit, within the oracle's 1e-4."""
    _torch()
    if decoder == "stepwise":
        monkeypatch.setenv("LVSR_NO_DEC_SCAN", "1")
    else:
        monkeypatch.delenv("LVSR_NO_DEC_SCAN", raising=False)
    cfg = O.make_config(prior=dict(type="window_around_median", before=5, after=7), energy_normalizer="logistic",
                        **PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    params[BIAS][:] = ENERGY_BIAS["logistic"]
    x, m, labels, lm = O.synthetic_batch(cfg, B=6, T=64, seed=21)
    import torch
    serial = _inference(make_recognizer(cfg, params), torch.cuda.default_stream(), x, m, labels, lm, delay=False)
    rec = make_recognizer(cfg, params)
    warm = _inference(rec, stream, x, m, labels, lm, delay=False)
    got = _inference(rec, stream, x, m, labels, lm, delay=True)
    for k in ("att", "attm", "P", "all", "cost", "gen"):
        assert _equal(warm[k], serial[k]) and _equal(got[k], serial[k]), k
    att, attm = O.encoder(cfg, params, x, m)
    want = O.cost_matrix(cfg, params, att, attm, labels, lm, return_all=True)
    assert rel_err(got["att"], att) < TOL
    for k in ("costs", "weights", "energies", "states", "weighted_averages"):
        assert rel_err(got["all"][k], want[k]) < TOL, k
    assert rel_err(got["cost"], want["costs"]) < TOL


def _utterances(cfg, seed=5):
    rng = np.random.RandomState(seed)
    return [rng.normal(size=(T, cfg["num_features"])).astype(np.float32) for T in (64, 37, 52, 45)]


def _search(rec, s, utts, delay, beam=5):
    rec.init_beam_search(beam)
    return _on(s, rec._beam_search.search_many, utts, rec.eos_label, [int(u.shape[0] / 3.0) for u in utts],
               raise_on_failure=False, delay=delay)


def test_beam_search_is_ordered_on_the_stream(stream):
    """search_many at beam 5 behind a queued spin: the serial answers, and the oracle's tokens where it finds any."""
    torch = _torch()
    cfg = O.make_config(max_decoded_length_scale=3.0, **PYRAMID)
    params = _peaky(cfg, 11)
    utts = _utterances(cfg)
    serial = _search(make_recognizer(cfg, params), torch.cuda.default_stream(), utts, delay=False)
    rec = make_recognizer(cfg, params)
    _search(rec, stream, utts, delay=False)
    got = _search(rec, stream, utts, delay=True)
    assert _equal(got, serial)
    found = 0
    for u, g in zip(utts, got):
        try:
            want = O.beam_search(cfg, params, u.astype(np.float64), 5, max_length=int(u.shape[0] / 3.0))
        except O.CandidateNotFoundError:
            assert g is None
            continue
        found += 1
        assert g[0] == want[0]
        assert np.allclose(g[1], want[1], rtol=1e-3, atol=5e-3)
    assert found >= 1


def test_fused_beam_search_is_ordered_on_the_stream(stream, lm_file):
    """search_many with the language model fused, behind a queued spin: the serial answers bit for bit."""
    torch = _torch()
    path, cmap, _ = lm_file
    cfg = O.make_config(max_decoded_length_scale=3.0, **PYRAMID)
    params = _peaky(cfg, 11)
    lm = dict(LO_DEFAULTS, weight=0.5, no_transition_cost=20.0, path=path)
    utts = _utterances(cfg)
    serial = _search(_recognizer(cfg, params, lm=lm, cmap=cmap), torch.cuda.default_stream(), utts, delay=False)
    rec = _recognizer(cfg, params, lm=lm, cmap=cmap)
    _search(rec, stream, utts, delay=False)
    got = _search(rec, stream, utts, delay=True)
    assert _equal(got, serial)
    assert any(g is not None for g in got)


# ---- training ----------------------------------------------------------------------------------------------------

def _train_setup(normalizer, seed=5):
    cfg = O.make_config(energy_normalizer=normalizer, **PYRAMID)
    params = O.init_params(cfg, seed=seed, scale=10.0)
    if normalizer != "softmax":
        params[BIAS][:] = ENERGY_BIAS[normalizer]
    return cfg, params


def _device_batch(s, batch):
    pkg = package()
    return dict(zip(pkg.GradientDescent.SOURCES, _dev(s, *batch)))


def _assert_params(got, ref, what):
    for k, v in ref.items():
        # the UPDATE is compared (new - old would cancel; the parameters themselves are O(0.1..1))
        assert np.abs(got[k] - v).max() <= 2e-5 * max(1.0, np.abs(v).max()) + 1e-6, (what, k, np.abs(got[k] - v).max())


def _warm_up(s, cfg, rec, algo, params, cost=False):
    """One update (and host cost) on s at the shapes the test uses, without a spin: it sizes the workspaces and
    allocates the optimizer state, which synchronise the stream.  Then the parameters and the optimizer state are put
    back, so the updates under test start from `params` and a fresh optimizer."""
    batch = O.synthetic_batch(cfg, B=4, T=40, seed=99)
    _on(s, algo.process_batch, _device_batch(s, batch), delay=False)
    if cost:
        _on(s, rec.cost, *batch, delay=False)
    rec.set_parameter_values(params)
    _on(s, algo.initialize, delay=False)


# momentum + AdaDelta + max-norm, the TIMIT main stage's rules, with a step that moves the energy bias by over 1e-2
TRAIN = G.make_train_config(gradient_threshold=100.0, rules=("momentum", "adadelta"), scale=5.0, momentum=0.5,
                            decay_rate=0.95, epsilon=1e-4, max_norm=1.0)


@pytest.mark.parametrize("normalizer", ["softmax", "logistic", "relu"])
def test_training_steps_are_ordered_on_the_stream(stream, normalizer):
    """A warm-up update undone by set_parameter_values and initialize(), then two updates each behind a queued spin;
    at once after each: the gradient norm and every parameter against G.train_step.  With logistic and relu the energy bias is a kernel argument read back after the
    update: the cost of the updated model (again behind a spin) must be the oracle's on the updated parameters."""
    _torch()
    pkg = package()
    cfg, params = _train_setup(normalizer)
    rec = make_recognizer(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(TRAIN, dict(max_norm=1.0)))
    algo.initialize()
    _warm_up(stream, cfg, rec, algo, params, cost=normalizer != "softmax")
    ref, state = OrderedDict((k, v.copy()) for k, v in params.items()), {}
    for step in range(2):
        batch = O.synthetic_batch(cfg, B=4, T=40, seed=100 + step)
        dbatch = _device_batch(stream, batch)
        old_bias = ref.get(BIAS)
        ref, ref_cost, ref_grads = G.train_step(cfg, ref, state, batch, TRAIN)
        _on(stream, algo.process_batch, dbatch)
        norm = algo.total_gradient_norm()
        got = rec.get_parameter_values()
        want_norm = G.l2_norm(ref_grads.values())
        assert abs(norm - want_norm) <= 1e-4 * want_norm, (step, norm, want_norm)
        _assert_params(got, ref, step)
        assert abs(float(algo.last_cost.item()) - ref_cost) <= 1e-4 * abs(ref_cost), (step, ref_cost)
        if normalizer != "softmax":
            assert abs(ref[BIAS][0] - old_bias[0]) >= 1e-2, (old_bias, ref[BIAS])    # a stale bias is visible
            x, m, labels, lm = batch
            cost = _on(stream, rec.cost, x, m, labels, lm)
            want = O.recognizer_cost(cfg, ref, x, m, labels, lm)
            assert rel_err(cost, want) < TOL, (step, rel_err(cost, want))


NOISE = dict(num_examples=1000, init_sigma=1e-2, model_cost_coefficient=0.5, seed=7)
NOISE_TRAIN = G.make_train_config(gradient_threshold=2.0, rules=("momentum", "adadelta"), scale=0.05, momentum=0.5,
                                  decay_rate=0.95, epsilon=1e-6, max_norm=1.0)


def _noise_algo(cfg, params):
    pkg = package()
    rec = make_recognizer(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(NOISE_TRAIN, dict(max_norm=1.0)),
                               adaptive_noise=NOISE)
    algo.initialize()
    return rec, algo


def _eps(algo, rec, s, update):
    """The noise of update `update` in the parameter layout (lvsr_train_noise_sample), drawn on s."""
    torch = _torch()
    pkg = package()
    buf = torch.zeros((algo._n,), dtype=torch.float32, device=rec.device)
    s.wait_stream(torch.cuda.default_stream())
    with torch.cuda.stream(s):
        pkg._lib.check(pkg._lib.load().lvsr_train_noise_sample(rec._require_ready(), update, buf.data_ptr(),
                                                               rec._stream()))
        flat = buf.cpu().numpy()
    shapes = rec.parameter_shapes()
    return {k: flat[o:o + c].reshape(shapes[k]).astype(np.float64) for k, (o, c) in algo._offsets().items()}


def _assert_noise(got_ls2, ls2, what):
    for k, w in ls2.items():
        assert np.abs(got_ls2[AN.noise_name(k)] - w).max() <= 1e-4 * np.abs(w).max(), (what, k)


def test_adaptive_noise_with_logistic_is_ordered_on_the_stream(stream):
    """A warm-up adaptive-noise update, then one behind a queued spin: at once after it, the means, the log-variances
    and the norm against adaptive_noise_oracle; then cost_and_gradients behind a spin against the oracle at the next
    update's noise."""
    _torch()
    cfg, params = _train_setup("logistic")
    rec, algo = _noise_algo(cfg, params)
    b0, batch = O.synthetic_batch(cfg, B=3, T=32, seed=24), O.synthetic_batch(cfg, B=3, T=32, seed=25)
    ref = {k: np.asarray(v, np.float32).astype(np.float64) for k, v in params.items()}
    ls2 = AN.init_ls2(ref, NOISE["init_sigma"])
    state = {}
    ref, ls2, _, _, _ = AN.train_step(cfg, ref, ls2, state, b0, NOISE_TRAIN, _eps(algo, rec, stream, 0),
                                      NOISE["num_examples"], NOISE["model_cost_coefficient"])
    _on(stream, algo.process_batch, _device_batch(stream, b0), delay=False)
    ref, ls2, cost, _, norm = AN.train_step(cfg, ref, ls2, state, batch, NOISE_TRAIN, _eps(algo, rec, stream, 1),
                                            NOISE["num_examples"], NOISE["model_cost_coefficient"])
    _on(stream, algo.process_batch, _device_batch(stream, batch))
    got_ls2 = algo.noise_parameter_values()
    got = rec.get_parameter_values()
    got_norm = algo.total_gradient_norm()
    _assert_noise(got_ls2, ls2, "update")
    for k, v in ref.items():
        assert np.abs(got[k] - v).max() <= 1e-4 * np.abs(v).max(), k
    assert abs(got_norm - norm) <= 1e-4 * norm, (got_norm, norm)
    assert abs(float(algo.last_cost.item()) - cost) <= 1e-4 * abs(cost)
    # the gradients at update 2's noise
    batch2 = O.synthetic_batch(cfg, B=3, T=32, seed=26)
    want_cost, gp, gl, _ = AN.cost_and_grads(cfg, ref, ls2, _eps(algo, rec, stream, 2), batch2, NOISE["num_examples"],
                                             NOISE["model_cost_coefficient"])
    got_cost, grads = _on(stream, algo.cost_and_gradients, _device_batch(stream, batch2))
    assert abs(got_cost - want_cost) <= 1e-4 * abs(want_cost), (got_cost, want_cost)
    for group, name in ((gp, lambda k: k), (gl, AN.noise_name)):
        gmax = max(np.abs(w).max() for w in group.values())
        for k, w in group.items():
            err = np.abs(grads[name(k)].astype(np.float64) - w).max()
            assert err <= 1e-4 * np.abs(w).max() + 1e-6 * gmax, (name(k), err, np.abs(w).max())


# ---- host calls wait for the work queued on the handle -------------------------------------------------------------

def test_set_parameter_values_waits_for_a_queued_cost(stream):
    """A cost_matrix queued behind a spin, then set_parameter_values at once: the queued cost is the old parameters'
    and the next one the new parameters', each bit-identical to a serial run.  A first cost_matrix of the same shape
    sizes the workspace, so that the queued one does not wait for the spin in Arena::reserve."""
    torch = _torch()
    cfg = O.make_config(**PYRAMID)
    old, new = O.init_params(cfg, seed=5, scale=10.0), O.init_params(cfg, seed=6, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=6, T=64, seed=21)
    att, attm = O.encoder(cfg, old, x, m)
    att, attm = att.astype(np.float32), attm.astype(np.float32)
    serial = [make_recognizer(cfg, p).cost_matrix(labels, lm, att, attm).cpu().numpy() for p in (old, new)]
    rec = make_recognizer(cfg, old)
    yd, ymd, ad, amd = _dev(stream, labels, lm, att, attm)
    warm = _on(stream, rec.cost_matrix, yd, ymd, ad, amd, delay=False)
    c_old = _on(stream, rec.cost_matrix, yd, ymd, ad, amd)
    rec.set_parameter_values(new)
    c_new = _on(stream, rec.cost_matrix, yd, ymd, ad, amd)
    stream.synchronize()
    assert np.array_equal(warm.cpu().numpy(), serial[0])
    assert np.array_equal(c_old.cpu().numpy(), serial[0])
    assert np.array_equal(c_new.cpu().numpy(), serial[1])
    torch.cuda.synchronize()


def test_optimizer_reset_waits_for_a_queued_step(stream):
    """After a warm-up step that is undone, a momentum step queued behind a spin, then GradientDescent.initialize()
    (lvsr_train_reset) at once: the next step is the oracle's step from a fresh optimizer state."""
    _torch()
    pkg = package()
    cfg, params = _train_setup("softmax")
    tc = G.make_train_config(gradient_threshold=100.0, rules=("momentum",), scale=0.5, momentum=0.9, max_norm=0.0)
    rec = make_recognizer(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(tc, {}))
    algo.initialize()
    _warm_up(stream, cfg, rec, algo, params)
    b1, b2 = (O.synthetic_batch(cfg, B=4, T=40, seed=100 + i) for i in range(2))
    ref, _, _ = G.train_step(cfg, params, {}, b1, tc)
    ref, _, grads = G.train_step(cfg, ref, {}, b2, tc)          # fresh optimizer state
    d1, d2 = _device_batch(stream, b1), _device_batch(stream, b2)
    _on(stream, algo.process_batch, d1)
    queued = (algo._buf, algo._cost)          # the queued step's own buffers stay alive until it has run
    _on(stream, algo.initialize, delay=False)
    _on(stream, algo.process_batch, d2)
    norm = algo.total_gradient_norm()
    got = rec.get_parameter_values()
    want_norm = G.l2_norm(grads.values())
    assert abs(norm - want_norm) <= 1e-4 * want_norm
    _assert_params(got, ref, "after the reset")
    del queued


def test_set_noise_parameter_values_waits_for_a_queued_step(stream):
    """After a warm-up update, an adaptive-noise update queued behind a spin, then set_noise_parameter_values at once:
    the values read back are the ones set, not the queued update's, and the next update is the oracle's from them."""
    _torch()
    cfg, params = _train_setup("logistic")
    rec, algo = _noise_algo(cfg, params)
    b0, b1, b2 = (O.synthetic_batch(cfg, B=3, T=32, seed=24 + i) for i in range(3))
    ref = {k: np.asarray(v, np.float32).astype(np.float64) for k, v in params.items()}
    ls2 = AN.init_ls2(ref, NOISE["init_sigma"])
    eps0, eps1, eps2 = (_eps(algo, rec, stream, u) for u in range(3))
    state = {}
    ref, ls2, _, _, _ = AN.train_step(cfg, ref, ls2, state, b0, NOISE_TRAIN, eps0, NOISE["num_examples"],
                                      NOISE["model_cost_coefficient"])
    ref, _, _, _, _ = AN.train_step(cfg, ref, ls2, state, b1, NOISE_TRAIN, eps1, NOISE["num_examples"],
                                    NOISE["model_cost_coefficient"])
    rng = np.random.RandomState(3)
    mine = OrderedDict((k, (np.float32(np.log(2e-2) * 2.0 / AN.LOG_SIGMA_SCALE) *
                            (1 + 0.1 * rng.uniform(size=np.shape(v)))).astype(np.float32)) for k, v in ref.items())
    _on(stream, algo.process_batch, _device_batch(stream, b0), delay=False)
    _on(stream, algo.process_batch, _device_batch(stream, b1))
    algo.set_noise_parameter_values({AN.noise_name(k): v for k, v in mine.items()})
    got = algo.noise_parameter_values()
    for k, v in mine.items():
        assert np.array_equal(got[AN.noise_name(k)], v), k
    ls2 = OrderedDict((k, v.astype(np.float64)) for k, v in mine.items())
    ref, ls2, cost, _, norm = AN.train_step(cfg, ref, ls2, state, b2, NOISE_TRAIN, eps2, NOISE["num_examples"],
                                            NOISE["model_cost_coefficient"])
    _on(stream, algo.process_batch, _device_batch(stream, b2))
    got_ls2 = algo.noise_parameter_values()
    got_norm = algo.total_gradient_norm()
    _assert_noise(got_ls2, ls2, "after the set")
    assert abs(got_norm - norm) <= 1e-4 * norm, (got_norm, norm)


# ---- one handle, two streams; two handles, two streams ---------------------------------------------------------------

def test_one_handle_two_streams_arena_growth():
    """After a warm-up encode on s1, an encode queued behind a spin on s1, then at once a larger encode on s2 of the
    same handle, which grows its workspace: both equal the serial results."""
    torch = _torch()
    s1, s2 = _side_stream(), _side_stream()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    small, large = O.synthetic_batch(cfg, B=2, T=32, seed=1), O.synthetic_batch(cfg, B=12, T=160, seed=2)
    base = make_recognizer(cfg, params)
    want = [[t.cpu().numpy() for t in base.encode(b[0], b[1])] for b in (small, large)]
    rec = make_recognizer(cfg, params)
    xs, ms = _dev(s1, small[0], small[1])
    xl, ml = _dev(s2, large[0], large[1])
    _on(s1, rec.encode, xs, ms, delay=False)
    a1 = _on(s1, rec.encode, xs, ms)
    a2 = _on(s2, rec.encode, xl, ml, delay=False)
    s1.synchronize()
    s2.synchronize()
    assert all(np.array_equal(g.cpu().numpy(), w) for g, w in zip(a1, want[0]))
    assert all(np.array_equal(g.cpu().numpy(), w) for g, w in zip(a2, want[1]))
    torch.cuda.synchronize()


def test_one_handle_two_streams_training_then_encode():
    """After a warm-up step on s1 and encode on s2, a training step queued behind a spin on s1, then at once an encode
    on s2: the encode runs on the updated parameters, as in a serial run."""
    torch = _torch()
    pkg = package()
    s1, s2 = _side_stream(), _side_stream()
    cfg, params = _train_setup("softmax")
    batches = [O.synthetic_batch(cfg, B=4, T=40, seed=100 + i) for i in range(2)]
    x, m = O.synthetic_batch(cfg, B=6, T=64, seed=3)[:2]

    def run(rec, algo, sa, sb, delay):
        d = [_device_batch(sa, b) for b in batches]
        xd, md = _dev(sb, x, m)
        out = []
        for i in range(2):                # the first round sizes the workspaces and allocates the optimizer state
            _on(sa, algo.process_batch, d[i], delay=delay and i > 0)
            out.append(_on(sb, rec.encode, xd, md, delay=False))
        sa.synchronize()
        sb.synchronize()
        return [t.cpu().numpy() for att in out for t in att]

    def fresh():
        rec = make_recognizer(cfg, params)
        algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(TRAIN, dict(max_norm=1.0)))
        algo.initialize()
        return rec, algo
    d = torch.cuda.default_stream()
    want = run(*fresh(), d, d, delay=False)
    got = run(*fresh(), s1, s2, delay=True)
    assert all(np.array_equal(g, w) for g, w in zip(got, want))


def test_two_handles_two_streams_interleaved():
    """Two models, each on its own stream and warmed up there, with their calls enqueued in turn behind spins: each
    equals its sequential run."""
    torch = _torch()
    s = [_side_stream(), _side_stream()]
    cfg = O.make_config(**PYRAMID)
    params = [O.init_params(cfg, seed=5 + i, scale=10.0) for i in range(2)]
    batches = [O.synthetic_batch(cfg, B=4 + 2 * i, T=48 + 16 * i, seed=30 + i) for i in range(2)]

    def sequential(i):
        rec = make_recognizer(cfg, params[i])
        x, m, y, ym = batches[i]
        att, attm = rec.encode(x, m)
        return [att.cpu().numpy(), rec.cost_matrix(y, ym, att, attm).cpu().numpy()]
    want = [sequential(i) for i in range(2)]
    recs = [make_recognizer(cfg, p) for p in params]
    dev = [_dev(s[i], *batches[i]) for i in range(2)]
    for i in range(2):
        att, attm = _on(s[i], recs[i].encode, dev[i][0], dev[i][1], delay=False)
        _on(s[i], recs[i].cost_matrix, dev[i][2], dev[i][3], att, attm, delay=False)
    enc = [_on(s[i], recs[i].encode, dev[i][0], dev[i][1]) for i in range(2)]
    costs = [_on(s[i], recs[i].cost_matrix, dev[i][2], dev[i][3], enc[i][0], enc[i][1]) for i in range(2)]
    for i in range(2):
        s[i].synchronize()
        assert np.array_equal(enc[i][0].cpu().numpy(), want[i][0])
        assert np.array_equal(costs[i].cpu().numpy(), want[i][1])
    torch.cuda.synchronize()
