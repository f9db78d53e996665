"""The training step against the float64 gradient oracle at long encoded lengths, up to the longest the attention
backward accepts, at the bar of test_gpu_train.py (helpers.check_grads: the cost to 1e-4, every parameter's gradient
to 1e-4 of its own largest entry plus a floor of 1e-6 of the model's largest).

att_bwd_kernel (csrc/train_kernels.cuh) runs two CTAs of 512 threads per utterance; several of its loops take a number
of passes that grows with the window length Tw, with T' or with conv_n, and at the short lengths of the other gradient
tests every one of them runs once.  Each case here names the branch it is for and asserts, from shape arithmetic or
from the oracle's forward weights, that it reaches it.  One or two utterances per case keep the oracle's autograd
tape under 2.5 GB; the oracle takes about 70 s of 8 CPU cores for the whole file, most of it in the three cases of
thousands of encoder steps (T'max, the benchmark's batch and content attention at 4400 frames)."""
import math

import numpy as np
import pytest

import bench
import content_oracle as CO
from helpers import O, check_grads, package

pytestmark = pytest.mark.gpu

# one unsubsampled BiGRU(128) layer: T' = T
ONE = dict(num_features=40, dims_bidir=[128], subsample=[1], dim_dec=128, dim_matcher=256, conv_n=8,
           conv_num_filters=10, num_phonemes=32, post_merge_dims=[128], maxout_pieces=2)
ATT = O._ATT + "/"

AB_NT, AB_CS, AB_TILE = 512, 2, 16       # threads per CTA, CTAs per utterance, positions per tile of att_bwd_kernel
SMEM_OPTIN_FLOATS = 227 * 1024 // 4      # the largest dynamic shared memory a CTA may opt in to on H100


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _att_bwd_smem_floats(M, E, K, n, tc_cap):
    """att_bwd_smem_floats (csrc/train_kernels.cuh), restated: the dynamic shared memory of att_bwd_kernel when a CTA
    owns up to tc_cap window positions."""
    KP = 12 if K <= 12 else 16
    return ((tc_cap + 2 * n + 8) + 4 + (2 * n + 1) * KP + K * M + 2 * tc_cap * KP + (tc_cap + 4) + AB_TILE * M + E
            + 64 + 16)


def _longest_trainable(M, E, K, n):
    """The longest T' whose att_bwd_kernel fits the opt-in shared memory: two CTAs of tc_cap = ceil(T' / 2)."""
    tc = 0
    while _att_bwd_smem_floats(M, E, K, n, tc + 1) <= SMEM_OPTIN_FLOATS:
        tc += 1
    return AB_CS * tc


def _passes(Tw, Tp, n):
    """The passes att_bwd_kernel's block-strided loops take for a window of Tw positions of T' = Tp, in the CTA that
    owns the larger half, nt = ceil(Tw / 2): the location features (4 lanes per position), the gradient of
    alpha_{i-1} (one thread per frame of T'), the staging of the alpha_{i-1} slice (nt + 2n + 8 values) and the
    filter gradient (2 lanes per tap)."""
    nt = -(-Tw // AB_CS)
    c = lambda x: -(-x // AB_NT)
    return dict(F=c(4 * nt), dA_out=c(Tp), salpha=c(nt + 2 * n + 8), dfilt=c(2 * (2 * n + 1)))


def _expanding_windows(cfg, Tp, L):
    """(begin, end) of the expanding prior at each of L steps, the oracle's own window arithmetic."""
    return [O.attention_window(cfg, Tp, None, np.array([i]))[:2] for i in range(L)]


def _weight_extents(cfg, params, batch):
    """(first, last + 1) of the positions with a non-zero weight at each step, over the batch, from the oracle's
    forward pass."""
    w = O.recognizer_cost(cfg, params, *batch, return_all=True)["weights"]        # [L, B, T']
    out = []
    for nz in (w > 0).any(axis=1):
        idx = np.flatnonzero(nz)
        out.append((int(idx[0]), int(idx[-1]) + 1) if idx.size else (0, 0))
    return out, w


def _batch(cfg, B, T, seed, L):
    """synthetic_batch with the label divisor that gives L label steps at T frames; its longest utterance is T."""
    batch = O.synthetic_batch(cfg, B=B, T=T, seed=seed, label_div=math.ceil(T / (L - 1)))
    assert batch[1].sum(axis=0).max() == T and batch[2].shape[0] == L
    return batch


# ---- pass boundaries of the conv backward over the full window --------------------------------------------------

@pytest.mark.parametrize("Tp,want", [(256, dict(F=1, dA_out=1, salpha=1)), (257, dict(F=2, dA_out=1, salpha=1)),
                                     (515, dict(F=3, dA_out=2, salpha=1)), (1030, dict(F=5, dA_out=3, salpha=2))],
                         ids=["256", "257", "515", "1030"])
def test_full_window_pass_boundaries(Tp, want):
    """The default prior attends the whole of T' at every step (Tw = T'): at 256 the location features take one pass,
    at 257 two; at 515 the gradient of alpha_{i-1} takes two passes, the location features three, and the window is
    odd so the two CTAs own 258 and 257 positions; at 1030 the alpha_{i-1} staging takes two passes too."""
    _torch()
    cfg = O.make_config(**ONE)
    params = O.init_params(cfg, seed=Tp, scale=10.0)
    batch = _batch(cfg, B=2, T=Tp, seed=Tp + 1, L=10)
    windows = _expanding_windows(cfg, Tp, 10)
    assert set(windows) == {(0, Tp)}
    got = _passes(Tp, Tp, cfg["conv_n"])
    assert {k: got[k] for k in want} == want, got
    print("T'=%d Tw=%d passes %s" % (Tp, Tp, got))
    check_grads(cfg, params, batch)


# ---- the longest T' the attention backward accepts --------------------------------------------------------------

def test_longest_encoded_length_trains_deterministically_and_one_more_frame_is_refused():
    """T'max = 3914 for ONE (K = 10 -> 12-float filter rows): 26 tc + 7228 floats <= 227 KiB gives tc = 1957 positions
    per CTA, so sF / sdF fill the opt-in shared memory.  At T'max the step matches the oracle, and a second call gives
    bit-identical gradients (the backward's reductions run in a fixed order).  At T'max + 1 the forward pass runs,
    training is refused before any kernel is launched, and the same handle then trains T'max again, bit for bit."""
    _torch()
    cfg = O.make_config(**ONE)
    M, E, K, n = cfg["dim_matcher"], O.dim_encoded(cfg), cfg["conv_num_filters"], cfg["conv_n"]
    tmax = _longest_trainable(M, E, K, n)
    assert _att_bwd_smem_floats(M, E, K, n, 1) == 26 + 7228
    assert tmax == 3914
    assert _att_bwd_smem_floats(M, E, K, n, tmax // 2) <= SMEM_OPTIN_FLOATS < _att_bwd_smem_floats(M, E, K, n, tmax // 2 + 1)
    print("T'max=%d: %d of %d shared-memory floats" % (tmax, _att_bwd_smem_floats(M, E, K, n, tmax // 2), SMEM_OPTIN_FLOATS))
    params = O.init_params(cfg, seed=11, scale=10.0)
    batch = _batch(cfg, B=1, T=tmax, seed=12, L=11)
    algo, rec = check_grads(cfg, params, batch)
    sources = lambda b: dict(zip(algo.SOURCES, b))
    cost, first = algo.cost_and_gradients(sources(batch))

    refused = _batch(cfg, B=1, T=tmax + 1, seed=13, L=11)
    assert np.isfinite(rec.cost(*refused)).all()                  # the forward pass takes this batch
    lib = package()._lib.load()
    lib.lvsr_launch_count(1)
    with pytest.raises((ValueError, RuntimeError)):
        algo.cost_and_gradients(sources(refused))
    assert lib.lvsr_launch_count(1) == 0

    cost2, again = algo.cost_and_gradients(sources(batch))
    assert cost2 == cost
    for k, g in first.items():
        assert np.array_equal(again[k], g), k


# ---- the benchmark's training batch -----------------------------------------------------------------------------

def test_two_utterances_of_the_benchmarked_training_batch():
    """bench.py --mode train's batch (WSJ architecture, M = E = 512, conv_n = 100, bench.init_values weights): its
    1500-frame utterance (T' = 375, 190 labels) and its shortest, at every label step.  The full window of 375
    positions gives nt = 188, so the location features take two passes; the 256-wide encoder runs the tensor-core
    scan with its tape and 1500 frames of BPTT."""
    _torch()
    cfg = O.make_config(**bench.NET)
    W = bench.TRAIN_WORKLOAD
    x, m, labels, lm = bench.synthetic_batch(**W, seed=bench.shard_seed(0, base=4321))
    lens = m.sum(axis=0)
    keep = [int(np.argmax(lens)), int(np.argmin(lens))]
    batch = (x[:, keep], m[:, keep], labels[:, keep], lm[:, keep])
    assert lens[keep[0]] == W["T"] and lm[:, keep].sum(axis=0)[0] == W["L"]
    print("utterances of %s frames, %s labels" % (lens[keep].astype(int).tolist(), lm[:, keep].sum(axis=0).astype(int).tolist()))
    Tp = 375
    assert set(_expanding_windows(cfg, Tp, W["L"])) == {(0, Tp)}
    assert _passes(Tp, Tp, cfg["conv_n"])["F"] == 2
    params = bench.init_values(O.param_shapes(cfg))
    _, rec = check_grads(cfg, params, batch)
    assert rec.encoded_length(W["T"]) == Tp
    plan = rec.encoder_plan()
    assert [p["bigru"] for p in plan] == ["mma"] * 4 and all(p["tape"] for p in plan), plan
    assert plan[0]["T"] == W["T"]


# ---- windows far from frame 0 -----------------------------------------------------------------------------------

def test_expanding_window_hundreds_of_frames_from_the_start():
    """An expanding prior that moves 20 to 120 frames a step at T' = 2000 with conv_n = 100: the window starts at
    frame 400 by step 20 and spans more than 1000 positions, so b0 is large in every offset of the backward (the
    alpha_{i-1} slice, P / dP / H rows, the gradient of alpha_{i-1}) while the location features take 7 passes and
    the staging 2."""
    _torch()
    prior = dict(type="expanding", initial_begin=0, initial_end=100, min_speed=20, max_speed=120)
    cfg = O.make_config(**dict(ONE, conv_n=100, prior=prior))
    params = O.init_params(cfg, seed=21, scale=10.0)
    batch = _batch(cfg, B=2, T=2000, seed=22, L=21)
    extents, _ = _weight_extents(cfg, params, batch)
    assert extents == _expanding_windows(cfg, 2000, 21)
    assert extents[20][0] == 400 and max(b for b, _ in extents) >= 300
    assert max(e - b for b, e in extents) > 1000
    widest = max(e - b for b, e in extents)
    print("windows %s, passes at the widest %s" % (extents[::5], _passes(widest, 2000, cfg["conv_n"])))
    check_grads(cfg, params, batch)


def test_window_around_median_at_a_timit_length():
    """window_around_median(100, 100) at T' = 2000 with conv_n = 100, the prior of the TIMIT-shaped recipe: each
    utterance's own window is masked inside the batch's cut.  With these random weights the cut drifts off frame 0
    (to [52, 340) by the last step) but stays in the first 400 frames, so this is not a far-window case."""
    _torch()
    prior = dict(type="window_around_median", before=100, after=100)
    cfg = O.make_config(**dict(ONE, conv_n=100, prior=prior))
    params = O.init_params(cfg, seed=24, scale=10.0)
    batch = _batch(cfg, B=2, T=2000, seed=24, L=21)
    extents, _ = _weight_extents(cfg, params, batch)
    print("windows", extents)
    assert max(b for b, _ in extents) > 0                         # the cut leaves frame 0
    assert max(e for _, e in extents) <= 400
    check_grads(cfg, params, batch)


# ---- wide and many filters at length ----------------------------------------------------------------------------

@pytest.mark.parametrize("net,kernel", [(dict(conv_n=128), "att_bwd_kernel<12>, 2 filter-gradient passes"),
                                        (dict(conv_num_filters=16), "att_bwd_kernel<16>")],
                         ids=["conv_n_128", "16_filters"])
def test_wide_and_many_filters_at_length(net, kernel):
    """conv_n = 128: 257 taps at 2 lanes each take two passes of the filter-gradient loop, and the alpha_{i-1} staging
    two; 16 filters: the kernel with 16-float filter rows.  Both over the full window at T' = 600."""
    _torch()
    cfg = O.make_config(**dict(ONE, **net))
    got = _passes(600, 600, cfg["conv_n"])
    if cfg["conv_n"] == 128:
        assert got["dfilt"] == 2 and got["salpha"] == 2, got
    else:
        assert cfg["conv_num_filters"] > 12
    print(kernel, got)
    params = O.init_params(cfg, seed=31, scale=10.0)
    check_grads(cfg, params, _batch(cfg, B=2, T=600, seed=32, L=11))


# ---- content attention past the conv limit ----------------------------------------------------------------------

def test_content_attention_beyond_the_conv_limit():
    """attention_type content at T' = 4400, which the conv model refuses to train: att_bwd_content_kernel with 2200
    positions per CTA, and 4400 steps of BPTT in each direction of the encoder."""
    _torch()
    cfg = CO.make_config(**ONE)
    assert _att_bwd_smem_floats(cfg["dim_matcher"], O.dim_encoded(cfg), cfg["conv_num_filters"], cfg["conv_n"],
                                2200) > SMEM_OPTIN_FLOATS
    params = CO.init_params(cfg, seed=41, scale=10.0)
    check_grads(cfg, params, _batch(cfg, B=1, T=4400, seed=42, L=12))


# ---- a one-position window --------------------------------------------------------------------------------------

def test_one_position_window():
    """An expanding prior of one position that never moves: Tw = 1, so the second CTA of each utterance owns no
    position and every weight is 1 on frame 0.  The attention parameters then get no gradient in the oracle, and the
    GPU's must be zero up to check_grads' floor."""
    _torch()
    from oracle import lvsr_oracle_grad as G
    prior = dict(type="expanding", initial_begin=0, initial_end=1, min_speed=0, max_speed=0)
    cfg = O.make_config(**dict(ONE, prior=prior))
    params = O.init_params(cfg, seed=51, scale=10.0)
    batch = _batch(cfg, B=2, T=64, seed=52, L=9)
    assert set(_expanding_windows(cfg, 64, 9)) == {(0, 1)}
    extents, w = _weight_extents(cfg, params, batch)
    assert set(extents) == {(0, 1)} and np.all(w[:, :, 0] == 1)
    _, want = G.cost_and_grads(cfg, params, *batch)
    att = [k for k in want if k.startswith(ATT)]
    assert len(att) == 6 and not any(want[k].any() for k in att)
    algo, _ = check_grads(cfg, params, batch)
    _, got = algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
    gmax = max(np.abs(v).max() for v in want.values())
    print("largest attention gradient / largest oracle gradient: %.1e" % (max(np.abs(got[k]).max() for k in att) / gmax))
