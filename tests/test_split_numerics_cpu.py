"""Numerics of the fp16 head/tail split the tensor-core BiGRU (csrc/bigru.cu: bigru_mma_kernel) feeds to the tensor cores,
restated in numpy: x = head + tail / 2^11 with fp16 head and fp16 tail, product
head_w*head_h + (head_w*tail_h + tail_w*head_h) / 2^11.  The claim in DESIGN.md section 2 is an error of 2^-21 of sum |w h|
(the dropped tail*tail term), i.e. the class of the 3xTF32 split; the power-of-two range scaling must be exact."""
import numpy as np

SCALE = 2048.0


def split(x):
    x = np.asarray(x, dtype=np.float32)
    head = x.astype(np.float16)
    tail = ((x - head.astype(np.float32)) * np.float32(SCALE)).astype(np.float16)
    return head, tail


def split_dot(w, h):
    """[K, N] x [K] -> [N] the way the kernels combine the three products (products and sums in float64: the tensor core's
    fp32 accumulation adds its own 2^-24 per term, which is not what is under test)."""
    wh, wt = split(w)
    hh, ht = split(h)
    wh, wt, hh, ht = (a.astype(np.float64) for a in (wh, wt, hh, ht))
    main = (wh * hh[:, None]).sum(0)
    cross = (wh * ht[:, None]).sum(0) + (wt * hh[:, None]).sum(0)
    return main + cross / SCALE


def range_scale(max_abs):
    """mirror of range_scale() in bigru.cu"""
    if not (16384.0 < max_abs < 3.0e38):
        return 1.0, 1.0
    e = int(np.floor(np.log2(max_abs)))
    return 2.0 ** -(e - 13), 2.0 ** (e - 13)


def test_representation_error_is_2_pow_minus_22():
    rng = np.random.RandomState(0)
    x = np.concatenate([rng.uniform(-1, 1, 20000), rng.normal(0, 0.05, 20000), rng.normal(0, 1e-3, 20000)]).astype(np.float32)
    head, tail = split(x)
    back = head.astype(np.float64) + tail.astype(np.float64) / SCALE
    rel = np.abs(back - x.astype(np.float64)) / np.maximum(np.abs(x.astype(np.float64)), 2.0 ** -14)
    assert rel.max() <= 2.0 ** -22 * 1.01, rel.max()


def test_split_product_matches_float64_to_2_pow_minus_20():
    rng = np.random.RandomState(1)
    K, N = 256, 192
    w = rng.normal(0, 0.08, (K, N)).astype(np.float32)            # orthogonal-init sized recurrent weights
    for h in (rng.uniform(-1, 1, K), np.tanh(rng.normal(0, 2, K)), rng.normal(0, 1e-2, K)):
        h = h.astype(np.float32)
        exact = (w.astype(np.float64) * h.astype(np.float64)[:, None]).sum(0)
        got = split_dot(w, h)
        bound = (np.abs(w.astype(np.float64)) * np.abs(h.astype(np.float64))[:, None]).sum(0)
        assert (np.abs(got - exact) / bound).max() < 2.0 ** -20


def test_range_scaling_is_exact_and_keeps_heads_finite():
    rng = np.random.RandomState(2)
    K, N = 256, 16
    w = rng.normal(0, 0.08, (K, N)).astype(np.float32)
    w[3, 5] = 1.0e5                                               # fp16 overflows at 65504
    w[17, 2] = -2.5e5
    h = rng.uniform(-1, 1, K).astype(np.float32)
    sc, inv = range_scale(float(np.abs(w).max()))
    assert sc * inv == 1.0 and np.abs(w).max() * sc <= 16384.0
    ws = w * np.float32(sc)
    assert np.array_equal(ws.astype(np.float64) * inv, w.astype(np.float64))        # power of two: exact
    head, _ = split(ws)
    assert np.isfinite(head.astype(np.float32)).all()
    exact = (w.astype(np.float64) * h.astype(np.float64)[:, None]).sum(0)
    got = split_dot(ws, h) * inv
    bound = (np.abs(w.astype(np.float64)) * np.abs(h.astype(np.float64))[:, None]).sum(0)
    assert (np.abs(got - exact) / bound).max() < 2.0 ** -20
    assert range_scale(0.5) == (1.0, 1.0) and range_scale(16384.0) == (1.0, 1.0)


def test_heads_and_tails_share_one_mma_through_the_n_columns():
    """bigru_mma_kernel puts the heads of the 4 batch rows into N columns 0..3 and their tails into columns 4..7, so
    A = head_w yields head*head and head*tail at once; lanes tq < 2 then add column n + 4 of the same accumulator."""
    rng = np.random.RandomState(3)
    K, M, RB = 32, 16, 4
    w = rng.normal(0, 0.1, (K, M)).astype(np.float32)
    h = rng.uniform(-1, 1, (RB, K)).astype(np.float32)
    wh, wt = (a.astype(np.float64) for a in split(w))
    hh, ht = (a.astype(np.float64) for a in split(h))
    B = np.concatenate([hh, ht], axis=0).T                        # [K, 8]
    c1 = wh.T @ B                                                 # [16, 8]: A = heads of the weights
    c2 = wt.T @ B                                                 # A = tails (columns 4..7 = tail*tail: ignored)
    got = c1[:, :RB] + (c1[:, RB:] + c2[:, :RB]) / SCALE
    want = np.stack([split_dot(w, h[r]) for r in range(RB)], axis=1)
    assert np.allclose(got, want, rtol=0, atol=1e-15)
