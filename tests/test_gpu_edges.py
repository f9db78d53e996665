"""Edge cases of the hot path on the GPU: ragged / degenerate shapes, every readout variant, and
the error behaviour of the C ABI.  Same bar as test_gpu_parity.py (1e-4 relative against the
float64 oracle, everything through ctypes -> liblvsr_b200.so)."""
import numpy as np
import pytest

from helpers import O, PYRAMID, SMALL, make_recognizer, package, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4
KEYS = ("costs", "weights", "energies", "states", "weighted_averages")


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _compare_cost(cfg, params, x, m, labels, lm, plan=None):
    """plan (optional): called with the encoder plan report of the forward."""
    want = O.recognizer_cost(cfg, params, x, m, labels, lm, return_all=True)
    rec = make_recognizer(cfg, params)
    att, attm = rec.encode(x, m)
    if plan is not None:
        plan(rec.encoder_plan())
    o_att, o_mask = O.encoder(cfg, params, x, m)
    assert rel_err(att.cpu().numpy(), o_att) < TOL
    assert np.array_equal(attm.cpu().numpy(), o_mask.astype(np.float32))
    got = rec.cost_matrix(labels, lm, att, attm, return_all=True)
    errs = {k: rel_err(got[k].cpu().numpy(), want[k]) for k in KEYS if k in want}
    for k, e in errs.items():
        assert e < TOL, (k, e)
    return errs


def test_very_short_utterances_in_a_long_batch():
    """Lengths 1, 2, 3 and 5 frames next to a full-length utterance: after the 4x pyramid some
    rows keep a single encoded frame; masked recurrences must carry the state through padding
    (B/bricks/recurrent.py:224-231 with mask) and the attention must put all weight on it."""
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=13, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=6, T=45, seed=5)
    lens = [1, 2, 3, 5, 45, 17]
    for b, n in enumerate(lens):
        m[:, b] = (np.arange(45) < n)
    x *= m[:, :, None]
    errs = _compare_cost(cfg, params, x, m, labels, lm)
    print("short utterances", errs)


@pytest.mark.parametrize("B,T", [(1, 9), (1, 64), (3, 8), (33, 21)])
def test_odd_batch_and_length_shapes(B, T):
    """Batches that do not fill a cluster's rows (1, 3), that spill into a second wave of row
    groups (33) and lengths that are not multiples of the subsampling product."""
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=2, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=B, T=T, seed=B * 100 + T, min_frac=0.3)
    _compare_cost(cfg, params, x, m, labels, lm)


def test_single_decoder_step_and_single_label():
    _torch()
    cfg = O.make_config(**SMALL)
    params = O.init_params(cfg, seed=4, scale=10.0)
    x, m, _, _ = O.synthetic_batch(cfg, B=4, T=20, seed=8)
    labels = np.full((1, 4), cfg["eos_label"], dtype=np.int64)
    lm = np.ones((1, 4))
    _compare_cost(cfg, params, x, m, labels, lm)


@pytest.mark.parametrize("activation", ["relu", "tanh", "maxout"])
@pytest.mark.parametrize("use_states", [True, False])
def test_readout_variants(activation, use_states):
    """post_merge activation x use_states_for_readout (lvsr/bricks/recognizer.py:259-279)."""
    _torch()
    net = dict(SMALL)
    net.pop("maxout_pieces")
    cfg = O.make_config(post_merge_activation=activation, use_states_for_readout=use_states,
                        maxout_pieces=2 if activation == "maxout" else 1, **net)
    params = O.init_params(cfg, seed=6, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=5, T=33, seed=9)
    _compare_cost(cfg, params, x, m, labels, lm)


@pytest.mark.parametrize("B,T", [(5, 40), (16, 160)])
def test_feature_width_not_a_multiple_of_4(B, T):
    """123 features (WSJ fbank + deltas + double deltas): the tensor-core GEMM needs a contraction that is a multiple of
    4, so the first layer's fork GEMM runs on FFMA tiles; at a small batch and at 2560 rows."""
    _torch()
    cfg = O.make_config(**dict(PYRAMID, num_features=123))
    params = O.init_params(cfg, seed=11, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=B, T=T, seed=B + T)

    def both_paths(plan):
        assert [p["proj"] for p in plan] == ["ffma", "tc", "tc"], plan
    _compare_cost(cfg, params, x, m, labels, lm, plan=both_paths)


def test_label_mask_freezes_states_after_the_end():
    """Rows whose labels have ended keep their last state and contribute zero cost
    (B/bricks/sequence_generators.py:311-319)."""
    torch = _torch()
    cfg = O.make_config(**SMALL)
    params = O.init_params(cfg, seed=7, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=7, T=48, seed=3, min_frac=0.2)
    rec = make_recognizer(cfg, params)
    att, attm = rec.encode(x, m)
    got = rec.cost_matrix(labels, lm, att, attm, return_all=True)
    states = got["states"].cpu().numpy()          # [L, B, C]
    costs = got["costs"].cpu().numpy()
    L = labels.shape[0]
    for b in range(labels.shape[1]):
        n = int(lm[:, b].sum())
        if n < L:
            assert np.all(costs[n:, b] == 0.0)
            assert np.array_equal(states[n:, b], np.broadcast_to(states[n, b], states[n:, b].shape))


def test_repeated_calls_are_bit_identical():
    """No atomics with run-dependent order anywhere on the path: two calls give the same bits."""
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=9, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=10, T=70, seed=12)
    rec = make_recognizer(cfg, params)
    a1, am = rec.encode(x, m)
    a2, _ = rec.encode(x, m)
    assert bool((a1 == a2).all())
    r1 = rec.cost_matrix(labels, lm, a1, am, return_all=True)
    r2 = rec.cost_matrix(labels, lm, a1, am, return_all=True)
    for k in KEYS:
        assert bool((r1[k] == r2[k]).all()), k


def test_shape_errors_are_reported_not_crashed():
    _torch()
    pkg = package()
    cfg = O.make_config(**SMALL)
    params = O.init_params(cfg, seed=1, scale=10.0)
    rec = make_recognizer(cfg, params)
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=16, seed=1)
    with pytest.raises((RuntimeError, ValueError)):
        rec.encode(x[:, :, :-1], m)                     # wrong feature width
    att, attm = rec.encode(x, m)
    bad = labels.copy()
    bad[0, 0] = cfg["num_phonemes"] + 5                   # label outside the vocabulary
    with pytest.raises((RuntimeError, ValueError)):
        rec.cost_matrix(bad, lm, att, attm)
    assert pkg is not None


def test_mismatched_argument_shapes_raise_value_error():
    """Every array handed to the C ABI is shape-checked on the host first (ADVICE r1: a mismatch
    used to read out of bounds)."""
    _torch()
    cfg = O.make_config(**SMALL)
    rec = make_recognizer(cfg, O.init_params(cfg, seed=1, scale=10.0))
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=16, seed=1)
    att, attm = rec.encode(x, m)
    with pytest.raises(ValueError):
        rec.cost(x[:, :, :-1], m, labels, lm)            # feature width
    with pytest.raises(ValueError):
        rec.cost(x, m[:-1], labels, lm)                  # recordings_mask length
    with pytest.raises(ValueError):
        rec.cost(x, m, labels[:, :-1], lm)               # labels batch
    with pytest.raises(ValueError):
        rec.cost(x, m, labels, lm[:-1])                  # labels_mask length
    with pytest.raises(ValueError):
        rec.encode(x, m[:, :-1])
    with pytest.raises(ValueError):
        rec.cost_matrix(labels, lm, att[:, :-1], attm)   # attended batch != labels batch
    with pytest.raises(ValueError):
        rec.cost_matrix(labels, lm, att[:, :, :-1], attm)
    with pytest.raises(ValueError):
        rec.cost_matrix(labels, lm, att, attm[:-1])
    with pytest.raises(ValueError):
        rec.cost_matrix(labels, lm[:, :-1], att, attm)
    got = rec.cost(x, m, labels, lm)                     # the handle still works afterwards
    assert np.isfinite(got).all()


def test_model_on_second_device_while_first_is_current():
    """A handle lives on the device that was current at creation; later calls run there whatever
    device the caller has current (per-device function attributes, DeviceGuard in api.cu)."""
    torch = _torch()
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    cfg = O.make_config(**SMALL)
    params = O.init_params(cfg, seed=1, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=16, seed=1)
    want = O.recognizer_cost(cfg, params, x, m, labels, lm)
    pkg = package()
    for dev in ("cuda:1", "cuda:0"):
        rec = pkg.SpeechRecognizer(
            input_dims={"recordings": 40}, input_num_chars={}, eos_label=cfg["eos_label"], num_phonemes=32,
            dim_dec=128, dims_bidir=[128], subsample=[1], conv_n=8, conv_num_filters=10,
            post_merge_dims=[128], post_merge_activation=pkg.Maxout(2), device=torch.device(dev))
        rec.set_parameter_values(params)
        torch.cuda.set_device(0)
        assert rel_err(rec.cost(x, m, labels, lm), want) < 1e-4
        att, attm = rec.encode(x, m)
        assert str(att.device) == dev
        assert rel_err(rec.cost_matrix(labels, lm, att, attm).cpu().numpy(), want) < 1e-4


# ---- the tensor-core BiGRU kernel (hidden size 256: bigru_mma_kernel in csrc/bigru.cu) -------------------------------
ENC256 = dict(PYRAMID, dims_bidir=[256, 256], subsample=[1, 2])
WSJ_ENC = dict(PYRAMID, dims_bidir=[256, 256, 256, 256], subsample=[1, 1, 2, 2])


@pytest.mark.parametrize("B,T", [(1, 9), (3, 8), (5, 33), (33, 21), (70, 12)])
def test_tensor_core_bigru_odd_shapes(B, T):
    """The mma.sync BiGRU kernel on batches that do not fill its 4-row clusters, that need 18 clusters (33 rows) or more
    clusters than the device holds at once (70 rows -> 36 clusters, two waves) and on lengths that are not multiples of
    the subsampling; ragged masks.  Same oracle bar as every other path."""
    _torch()
    cfg = O.make_config(**ENC256)
    params = O.init_params(cfg, seed=4, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=B, T=T, seed=B * 10 + T, min_frac=0.2)
    if B >= 3:
        m[:, 0] = (np.arange(T) < 1)          # a one-frame utterance
        x *= m[:, :, None]
    _compare_cost(cfg, params, x, m, labels, lm)


def test_tensor_core_bigru_agrees_with_the_fp32_kernel(monkeypatch):
    """fp16 head/tail operands must reproduce the FFMA kernel to fp32 round-off at the metric batch (the split drops
    terms of 2^-22 only): run both kernels of csrc/bigru.cu on the same input."""
    torch = _torch()
    cfg = O.make_config(**WSJ_ENC)
    params = O.init_params(cfg, seed=9, scale=10.0)
    x, m, _, _ = O.synthetic_batch(cfg, B=64, T=200, seed=77, dtype=np.float32)
    rec = make_recognizer(cfg, params)
    monkeypatch.setenv("LVSR_BIGRU_MMA", "0")
    ref = rec.encode(x, m)[0].clone()
    assert [p["bigru"] for p in rec.encoder_plan()] == ["ffma"] * 4
    monkeypatch.setenv("LVSR_BIGRU_MMA", "1")
    got = rec.encode(x, m)[0]
    assert [p["bigru"] for p in rec.encoder_plan()] == ["mma"] * 4
    err = float((got - ref).abs().max() / ref.abs().max())
    print("mma vs ffma bigru", err)
    assert bool(torch.isfinite(got).all()) and err < 1e-5


def test_recurrent_weights_beyond_the_fp16_range():
    """A recurrent weight of 1e5 (fp16 overflows at 65504): the tensor-core kernel rescales a tile's fragments by a power
    of two, so the result is the fp32 kernel's -- the unit saturates, everything else keeps its accuracy."""
    _torch()
    cfg = O.make_config(**ENC256)
    params = O.init_params(cfg, seed=6, scale=10.0)
    for name in sorted(params):
        if name.endswith("gatedrecurrent.state_to_state") or name.endswith("gatedrecurrent.state_to_gates"):
            w = np.array(params[name])
            w[3, 5] = 1.0e5
            w[17, w.shape[1] - 2] = -2.5e5
            params[name] = w
    x, m, labels, lm = O.synthetic_batch(cfg, B=4, T=24, seed=21)
    _compare_cost(cfg, params, x, m, labels, lm)

