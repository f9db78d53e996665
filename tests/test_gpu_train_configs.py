"""The training step's gradients across the configurations lvsr accepts, against the float64 gradient oracle
(oracle/lvsr_oracle_grad.py), at the bar of test_gpu_train.py: the cost to 1e-4, every parameter's gradient to 1e-4 of
its own largest entry plus a floor of 1e-6 of the model's largest.  Small batches keep the oracle quick; the sweep
covers the branches of the backward kernels the architectures of test_gpu_train.py leave out: every readout
activation with and without the states in the readout, the window prior, 1 and 16 attention filters, vocabularies of
63 and 128, encoder stacks of other widths and subsampling, a feature width that is not a multiple of 4, and batch
edges.  Shapes the forward pass accepts and the backward kernels cannot take are refused on the host."""
import numpy as np
import pytest

from helpers import O, PYRAMID, check_grads, make_recognizer, package, relu_readout_kinks

pytestmark = pytest.mark.gpu


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _check(seed=5, B=4, T=48, **net):
    _torch()
    cfg = O.make_config(**dict(PYRAMID, **net))
    params = O.init_params(cfg, seed=seed, scale=10.0)
    batch = O.synthetic_batch(cfg, B=B, T=T, seed=seed + 20)
    return check_grads(cfg, params, batch)


@pytest.mark.parametrize("activation", ["tanh", "relu", "identity", "maxout"])
@pytest.mark.parametrize("use_states", [True, False], ids=["states", "no_states"])
def test_readout_activation_and_states(activation, use_states):
    """readout_bwd_kernel's Tanh / Rectifier / Identity / Maxout(2) branches; without the states in the readout
    (lvsr/bricks/recognizer.py:259-279) transform_states does not exist and the readout sends no gradient to s_{i-1}."""
    _check(post_merge_activation=activation, use_states_for_readout=use_states)


def test_window_around_mean_prior():
    """The window around the mean of the previous alignment (lvsr/bricks/attention.py:135-149) in the backward loop."""
    _check(prior=dict(type="window_around_mean", before=5, after=7))


@pytest.mark.parametrize("K", [1, 16])
def test_attention_filter_counts_with_short_filters(K):
    """att_bwd_kernel<12> with one filter (the reference's default conv_num_filters) and att_bwd_kernel<16> with 16,
    both with filters of length 2 * 2 + 1."""
    _check(conv_num_filters=K, conv_n=2)


@pytest.mark.parametrize("V", [63, 128])
def test_vocabulary_sizes(V):
    """V = 63 and V = 128, the largest vocabulary readout_bwd_kernel holds (four logits per lane)."""
    _check(num_phonemes=V)


@pytest.mark.parametrize("dims,subsample", [([128], [1]), ([256, 128], [1, 2]), ([128, 256], [1, 2]),
                                            ([128, 128, 128], [1, 3, 2])],
                         ids=["single_layer", "256_then_128", "128_then_256", "subsample_3"])
def test_encoder_stacks(dims, subsample):
    """One unsubsampled layer; mixed widths, which change Din of the input-gradient GEMM of the upper layer; a
    subsampling factor of 3."""
    _check(dims_bidir=dims, subsample=subsample)


def test_feature_width_not_a_multiple_of_4():
    """123 features (WSJ fbank + deltas + double deltas): the first layer's fork GEMMs run on FFMA tiles."""
    _, rec = _check(num_features=123)
    assert [p["proj"] for p in rec.encoder_plan()] == ["ffma", "tc", "tc"]


def test_odd_batch_with_a_one_frame_utterance():
    """B = 33 leaves a partial 4-row group in the BiGRU backward kernel; one utterance is a single frame long."""
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=8, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=33, T=24, seed=31)
    short = int(np.argmin(m.sum(axis=0)))                  # never the utterance synthetic_batch made full length
    m[:, short] = np.arange(24) < 1
    x *= m[:, :, None]
    assert m.sum(axis=0).max() == 24 and m.sum(axis=0).min() == 1
    check_grads(cfg, params, (x, m, labels, lm))


def test_single_label():
    """L = 1: one decoder step, the backward loop runs once and starts from the initial state."""
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=9, scale=10.0)
    x, m, _, _ = O.synthetic_batch(cfg, B=4, T=20, seed=4)
    labels = np.full((1, 4), cfg["eos_label"], dtype=np.int64)
    check_grads(cfg, params, (x, m, labels, np.ones((1, 4))))


@pytest.mark.parametrize("seed", [25, 26])
def test_tensor_core_backward_gemms_with_relu_readout_and_123_features(seed):
    """T * B = 2048 rows: the encoder's weight- and input-gradient GEMMs run on the tensor cores, here with a first layer
    of 123 inputs (a weight-gradient GEMM of 123 output rows) and the Rectifier readout.  In the batch of seed 25, the
    readout pre-activation of unit 74 at step 6 of utterance 31 is -2.5e-8 in float64, so the float32 forward may put it on
    either side of the Rectifier's kink (the tensor-core path gives +6e-7): check_grads compares that unit with the
    oracle's derivative from each side, everything at the unchanged tolerance."""
    _torch()
    cfg = O.make_config(**dict(PYRAMID, post_merge_activation="relu", num_features=123))
    params = O.init_params(cfg, seed=5, scale=10.0)
    batch = O.synthetic_batch(cfg, B=32, T=64, seed=seed)
    if seed == 25:
        assert (6, 31, 74) in relu_readout_kinks(cfg, params, batch)[0]
    check_grads(cfg, params, batch)


# ---- refusals -----------------------------------------------------------------------------------------------------

def test_vocabulary_and_matcher_beyond_the_kernels_are_refused():
    """129 symbols and a dim_matcher that is not a multiple of 128 are refused when the model is created, so neither the
    forward pass nor the training step ever sees them."""
    _torch()
    for net in (dict(num_phonemes=129), dict(dim_matcher=192)):
        cfg = O.make_config(**dict(PYRAMID, **net))
        with pytest.raises((ValueError, RuntimeError)):
            make_recognizer(cfg, O.init_params(cfg, seed=1, scale=10.0))


def _refuses_training_then_still_works(cfg, params, refused, accepted):
    pkg = package()
    rec = make_recognizer(cfg, params)
    assert np.isfinite(rec.cost(*refused)).all()                  # the forward pass takes this batch
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
    with pytest.raises((ValueError, RuntimeError)):
        algo.cost_and_gradients(dict(zip(algo.SOURCES, refused)))
    want = O.recognizer_cost(cfg, params, *accepted)
    got = rec.cost(*accepted)
    assert np.abs(got - want).max() <= 1e-4 * np.abs(want).max()
    return rec, algo


def test_post_merge_too_wide_for_the_readout_backward_is_refused():
    """A 1536-wide Tanh readout fits the forward readout kernel (8 rows x 1536 floats of shared memory) but not the
    backward one, which also holds 128 logits per row: training refuses it before running anything."""
    _torch()
    cfg = O.make_config(**dict(PYRAMID, post_merge_dims=[1536], post_merge_activation="tanh"))
    params = O.init_params(cfg, seed=3, scale=10.0)
    batch = O.synthetic_batch(cfg, B=3, T=32, seed=6)
    _refuses_training_then_still_works(cfg, params, batch, batch)


def test_utterance_too_long_for_the_attention_backward_is_refused():
    """4400 encoded frames: the forward attention spreads them over a cluster of CTAs, the backward kernel's two CTAs per
    utterance cannot hold its window in shared memory.  Training refuses the batch; a short batch still trains."""
    _torch()
    net = dict(PYRAMID, dims_bidir=[128], subsample=[1])
    cfg = O.make_config(**net)
    params = O.init_params(cfg, seed=3, scale=10.0)
    long_batch = O.synthetic_batch(cfg, B=1, T=4400, seed=6, label_div=400)
    short = O.synthetic_batch(cfg, B=3, T=32, seed=7)
    rec, algo = _refuses_training_then_still_works(cfg, params, long_batch, short)
    cost, _ = algo.cost_and_gradients(dict(zip(algo.SOURCES, short)))
    assert abs(cost - float(O.recognizer_cost(cfg, params, *short).sum() / 3)) <= 1e-4 * abs(cost)
