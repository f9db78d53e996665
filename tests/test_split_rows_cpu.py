"""The operand layout of the 8-row tensor-core BiGRU (csrc/bigru.cu: bigru_mma_kernel<D, TAPE, 8>), restated in numpy
lane by lane: the sender's 16-byte words [head01 head23 tail01 tail23] per 4-unit group, the receiving lane's one 16-byte
load per k-step, the B fragments of mma.sync m16n8k16 it yields, the three products head_w*H_head, head_w*H_tail and
tail_w*H_head, and the C fragment each lane stores.  The result must be head*head + (head*tail + tail*head) / 2^11 of
every (weight column, batch row): the numerics of the 4-row kernel (test_split_numerics_cpu.py)."""
import numpy as np

SCALE = 2048.0
RB, K, M = 8, 64, 16      # 8 batch rows, 4 k-steps, one M tile


def split(x):
    x = np.asarray(x, dtype=np.float32)
    head = x.astype(np.float16)
    tail = ((x - head.astype(np.float32)) * np.float32(SCALE)).astype(np.float16)
    return head, tail


def pack(lo, hi):
    """two fp16 values -> one 32-bit word, lower half = lower k index (split_pair)"""
    return np.uint32(np.float16(lo).view(np.uint16)) | (np.uint32(np.float16(hi).view(np.uint16)) << np.uint32(16))


def unpack(word):
    w = np.uint32(word)
    return (np.uint16(w & np.uint32(0xFFFF)).view(np.float16).astype(np.float64),
            np.uint16(w >> np.uint32(16)).view(np.float16).astype(np.float64))


def plane(h):
    """[RB, K] fp32 state -> [RB, K] words of one plane row: group u/4 holds (head01, head23, tail01, tail23), the order in
    which the elementwise thread of a role ships make_uint4(w0, w2, w1, w3)"""
    hh, ht = split(h)
    words = np.zeros((RB, K), np.uint32)
    for r in range(RB):
        for u in range(0, K, 4):
            words[r, u:u + 4] = [pack(hh[r, u], hh[r, u + 1]), pack(hh[r, u + 2], hh[r, u + 3]),
                                 pack(ht[r, u], ht[r, u + 1]), pack(ht[r, u + 2], ht[r, u + 3])]
    return words


def mma(a, b):
    """m16n8k16: a [16, 16], b [16, 8] -> [16, 8] (float64: the accumulation order is not under test)"""
    return a @ b


def test_three_products_over_the_interleaved_plane_match_the_split_dot():
    rng = np.random.RandomState(5)
    w = rng.normal(0, 0.1, (K, M)).astype(np.float32)          # [k, weight column]
    h = rng.uniform(-1, 1, (RB, K)).astype(np.float32)
    wh, wt = (a.astype(np.float64) for a in split(w))
    words = plane(h)

    # MMA k index kk of k-step ks <-> unit 16 ks + 4 (kk/2 % 4) + 2 (kk/8) + kk % 2 (the A fragments use the same order)
    def unit(ks, kk):
        return 16 * ks + 4 * ((kk // 2) % 4) + 2 * (kk // 8) + kk % 2

    acc = {t: np.zeros((M, RB)) for t in ("hh", "ht", "th")}
    for ks in range(K // 16):
        a_head = np.array([[wh[unit(ks, kk), mrow] for kk in range(16)] for mrow in range(M)])
        a_tail = np.array([[wt[unit(ks, kk), mrow] for kk in range(16)] for mrow in range(M)])
        b_head, b_tail = np.zeros((16, 8)), np.zeros((16, 8))
        for lane in range(32):
            g, tq = lane >> 2, lane & 3
            v = words[g, 16 * ks + 4 * tq:16 * ks + 4 * tq + 4]     # the lane's one 16-byte load
            # b0 = B[2 tq, 2 tq + 1][g], b1 = B[2 tq + 8, 2 tq + 9][g]; heads in v.x, v.y and tails in v.z, v.w
            b_head[2 * tq:2 * tq + 2, g] = unpack(v[0])
            b_head[2 * tq + 8:2 * tq + 10, g] = unpack(v[1])
            b_tail[2 * tq:2 * tq + 2, g] = unpack(v[2])
            b_tail[2 * tq + 8:2 * tq + 10, g] = unpack(v[3])
        acc["hh"] += mma(a_head, b_head)
        acc["ht"] += mma(a_head, b_tail)
        acc["th"] += mma(a_tail, b_head)

    # C fragment of lane (g, tq): c0, c1 = (column g, rows 2 tq, 2 tq + 1), c2, c3 = (column g + 8, same rows); all three
    # accumulators share it, so each lane combines its own registers and stores (column, row) pairs
    red = np.full((RB, M), np.nan)
    for lane in range(32):
        g, tq = lane >> 2, lane & 3
        for i, (mrow, r) in enumerate([(g, 2 * tq), (g, 2 * tq + 1), (g + 8, 2 * tq), (g + 8, 2 * tq + 1)]):
            red[r, mrow] = acc["hh"][mrow, r] + (acc["ht"][mrow, r] + acc["th"][mrow, r]) / SCALE
    assert not np.isnan(red).any()

    hh, ht = (a.astype(np.float64) for a in split(h))
    want = (hh @ wh) + ((ht @ wh) + (hh @ wt)) / SCALE             # [RB, M]
    assert np.allclose(red, want, rtol=0, atol=1e-13)
    exact = h.astype(np.float64) @ w.astype(np.float64)
    bound = np.abs(h.astype(np.float64)) @ np.abs(w.astype(np.float64))
    assert (np.abs(red - exact) / bound).max() < 2.0 ** -20


def test_a_load_phase_of_eight_lanes_covers_every_bank_once():
    """A 16-byte shared-memory load is served 8 lanes at a time.  Lanes 8q .. 8q + 7 read rows 2q and 2q + 1 at the same
    k-step; with a row stride of D + 16 words the two rows fall on different halves of the 32 banks."""
    D = 256
    rsh = D + 16
    for ks in range(D // 16):
        for q in range(4):
            banks = []
            for lane in range(8 * q, 8 * q + 8):
                g, tq = lane >> 2, lane & 3
                w0 = g * rsh + 16 * ks + 4 * tq
                banks += [(w0 + i) % 32 for i in range(4)]
            assert sorted(banks) == list(range(32)), (ks, q)
