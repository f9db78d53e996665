"""A numpy restatement of the training step's random draws -- TEST INFRASTRUCTURE ONLY.

The library draws dropout masks, weight-noise eps and adaptive-noise eps from Philox-4x32-10 (Salmon et al. 2011,
"Parallel random numbers: as easy as 1, 2, 3"; the generator of Random123 and of curand's curand_Philox4x32_10),
keyed by the 64-bit seed and countered by (position, update, stream tag).  This module computes the same draws on
the CPU from that definition alone, so the GPU's draws can be checked element by element rather than statistically:

  * dropout multiplier of element (t, b, f) of a [T, B, F] batch: 2 * bit (f % 32) of word (f / 32) % 4 of
    Philox(ctr = (t, utt_offset + b, update lo, 0xD0 << 24 | f / 128), key = seed), so 0 or 2 (mask / (1 - p),
    p = 0.5).  Only the low word of the update counter enters.
  * eps of flat element i: element i % 4 of the four normals of Philox(ctr = (q lo, q hi, update lo, update hi ^ tag),
    key = seed), q = i / 4, tag 0x57 << 24 for weight noise and 0 for adaptive noise.  The four words (x, y, z, w)
    give two Box-Muller pairs (x, y) -> eps 4q, 4q+1 and (z, w) -> 4q+2, 4q+3:
        u = float32((x >> 8) + 0.5) / 2^24,  v = (y >> 8) / 2^24,
        r = sqrt(-2 log u),  (r cos 2 pi v, r sin 2 pi v).
    u is formed as the device forms it: for x >> 8 >= 2^23 the half does not fit a float32 significand and the sum
    rounds to even, so u can be 1 (then r = 0).  The rest is computed here in float64.

Counters are uint64 numpy arrays holding 32-bit words; every function is vectorised over them.
"""
import numpy as np

M32 = np.uint64(0xFFFFFFFF)
PHILOX_M0, PHILOX_M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
PHILOX_W0, PHILOX_W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)

TAG_ADAPTIVE, TAG_WEIGHT_NOISE, TAG_DROPOUT = 0, 0x57 << 24, 0xD0 << 24
PARAM_ALIGN = 64          # every parameter's flat span starts at a multiple of 64 elements


def _u64(x):
    return np.asarray(x, dtype=np.uint64) & M32


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox-4x32-10 of counters (c0, c1, c2, c3) under keys (k0, k1): the four output words, uint64 arrays of
    32-bit values (broadcast over the inputs)."""
    c0, c1, c2, c3, k0, k1 = np.broadcast_arrays(*(_u64(a) for a in (c0, c1, c2, c3, k0, k1)))
    c0, c1, c2, c3, k0, k1 = (a.copy() for a in (c0, c1, c2, c3, k0, k1))
    for rnd in range(10):
        if rnd:
            k0 = (k0 + PHILOX_W0) & M32
            k1 = (k1 + PHILOX_W1) & M32
        p0 = PHILOX_M0 * c0                      # < 2^64: exact in uint64
        p1 = PHILOX_M1 * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32
    return c0, c1, c2, c3


def _key(seed):
    seed = int(seed)
    return seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF


def dropout_multiplier(seed, update, utt_offset, T, B, F):
    """The dropout multiplier {0, 2} of a [T, B, F] batch whose first utterance has global index utt_offset, as a
    float32 array."""
    words = (F + 127) // 128
    t = np.arange(T, dtype=np.uint64)[:, None, None]
    b = np.arange(B, dtype=np.uint64)[None, :, None] + np.uint64(utt_offset)
    hi = np.arange(words, dtype=np.uint64)[None, None, :] | np.uint64(TAG_DROPOUT)
    k0, k1 = _key(seed)
    w = np.stack(philox4x32_10(t, b, int(update) & 0xFFFFFFFF, hi, k0, k1), axis=-1)     # [T, B, words, 4]
    f = np.arange(F)
    word = w[:, :, f >> 7, (f >> 5) & 3]                                                  # [T, B, F]
    bit = (word >> (f & 31).astype(np.uint64)) & np.uint64(1)
    return (2.0 * bit).astype(np.float32)


def uniform_u(x):
    """u of Box-Muller from a 32-bit word, in (0, 1], rounded as float32((x >> 8) + 0.5) is."""
    top = (_u64(x) >> np.uint64(8)).astype(np.float32)
    return (top + np.float32(0.5)).astype(np.float64) / 2.0 ** 24


def uniform_v(y):
    return (_u64(y) >> np.uint64(8)).astype(np.float64) / 2.0 ** 24


def box_muller(x, y):
    """(r cos 2 pi v, r sin 2 pi v, r) in float64 from the words x (u) and y (v)."""
    r = np.sqrt(-2.0 * np.log(uniform_u(x)))
    v = uniform_v(y)
    return r * np.cos(2.0 * np.pi * v), r * np.sin(2.0 * np.pi * v), r


def eps_groups(seed, update, q, tag):
    """(eps [len(q), 4], r [len(q), 4]) of the flat groups q (elements 4q .. 4q+3) under stream tag `tag`: the
    normals and the Box-Muller radius each was scaled by."""
    q = np.asarray(q, dtype=np.uint64)
    update = int(update)
    k0, k1 = _key(seed)
    x, y, z, w = philox4x32_10(q & M32, q >> np.uint64(32), update & 0xFFFFFFFF,
                               ((update >> 32) & 0xFFFFFFFF) ^ tag, k0, k1)
    a0, a1, ra = box_muller(x, y)
    b0, b1, rb = box_muller(z, w)
    return np.stack([a0, a1, b0, b1], axis=1), np.stack([ra, ra, rb, rb], axis=1)


def flat_layout(counts):
    """[(offset, count)] of parameters of `counts` elements laid out one after another, each starting at a multiple
    of PARAM_ALIGN, and the flat length."""
    out, total = [], 0
    for c in counts:
        out.append((total, int(c)))
        total += -(-int(c) // PARAM_ALIGN) * PARAM_ALIGN
    return out, total


def _flat_eps(seed, update, spans, n, tag, subject=None):
    eps, rad = np.zeros(n), np.zeros(n)
    for i, (o, c) in enumerate(spans):
        if subject is not None and not subject[i]:
            continue
        g = (c + 3) // 4
        e, r = eps_groups(seed, update, np.arange(o // 4, o // 4 + g, dtype=np.uint64), tag)
        eps[o:o + c] = e.reshape(-1)[:c]
        rad[o:o + c] = r.reshape(-1)[:c]
    return eps, rad


def weight_noise_eps(seed, update, spans, n, subject):
    """(eps, r) of weight noise over a flat buffer of n elements: the normals on the spans [(offset, count)] whose
    `subject` flag is set, 0 on the other spans and on the padding between spans; r the Box-Muller radius of each
    (0 where eps is)."""
    return _flat_eps(seed, update, spans, n, TAG_WEIGHT_NOISE, subject)


def adaptive_noise_eps(seed, update, spans, n):
    """(eps, r) of adaptive weight noise: the normals on every span, 0 on the padding."""
    return _flat_eps(seed, update, spans, n, TAG_ADAPTIVE)


def eps_bar(r):
    """Absolute bound on |float32 eps - float64 eps| for Box-Muller radius r, both from the same words.  The device
    computes r c = sqrtf(-2 logf(u)) * cospif(2 v) (no fast math): logf and cospif/sinpif within 1 ulp, sqrtf and the
    product correctly rounded, -2 * and 2 * exact.  The relative errors add to at most (1/2 + 1/2 + 1 + 1/2) ulp of a
    float32 result; four ulps (2^-21) of max(r, 1) covers that with room, and the max(., 1) absorbs cancellation near
    the zeros of sin and cos."""
    return 4.0 * 2.0 ** -23 * np.maximum(np.asarray(r, dtype=np.float64), 1.0)
