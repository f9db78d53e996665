"""The numpy restatement of the training step's draws (tests/draws_oracle.py): Philox-4x32-10 against Random123's
published known-answer vectors, the dropout bit layout, Box-Muller, the flat layout the eps are keyed by, and the
stream tags that keep dropout, weight noise and adaptive noise apart."""
import numpy as np
import pytest

import content_oracle as CO
import draws_oracle as D
import regularization_oracle as RO
from helpers import O

# Random123 kat_vectors: philox4x32 10 (ctr, key, output)
KAT = [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
]


@pytest.mark.parametrize("ctr,key,want", KAT, ids=["zeros", "ones", "pi"])
def test_philox_known_answers(ctr, key, want):
    got = D.philox4x32_10(*ctr, *key)
    assert tuple(int(w) for w in got) == want


def test_philox_is_elementwise_over_arrays():
    """The vectorised form gives each lane what the scalar form gives it."""
    c0 = np.array([0, 0xffffffff, 0x243f6a88], dtype=np.uint64)
    c1 = np.array([0, 0xffffffff, 0x85a308d3], dtype=np.uint64)
    c2 = np.array([0, 0xffffffff, 0x13198a2e], dtype=np.uint64)
    c3 = np.array([0, 0xffffffff, 0x03707344], dtype=np.uint64)
    k0 = np.array([0, 0xffffffff, 0xa4093822], dtype=np.uint64)
    k1 = np.array([0, 0xffffffff, 0x299f31d0], dtype=np.uint64)
    words = np.stack(D.philox4x32_10(c0, c1, c2, c3, k0, k1), axis=1)
    assert [tuple(int(w) for w in row) for row in words] == [k[2] for k in KAT]


def test_dropout_multiplier_takes_bit_f_mod_32_of_word_f_div_32_mod_4_of_the_draw_of_f_div_128():
    seed, update, off, T, B, F = 0x0000000500000003, 7, 11, 3, 2, 300
    m = D.dropout_multiplier(seed, update, off, T, B, F)
    assert m.shape == (T, B, F) and m.dtype == np.float32 and set(np.unique(m)) <= {0.0, 2.0}
    for t, b, f in [(0, 0, 0), (2, 1, 31), (1, 0, 32), (1, 1, 127), (0, 1, 128), (2, 0, 200), (2, 1, 299)]:
        w = D.philox4x32_10(t, off + b, update, D.TAG_DROPOUT | (f >> 7), seed & 0xffffffff, seed >> 32)
        assert m[t, b, f] == 2.0 * ((int(w[(f >> 5) & 3]) >> (f & 31)) & 1), (t, b, f)
    # a shard at offset off + 1 draws column 1; the low word of the update alone keys the mask
    assert np.array_equal(D.dropout_multiplier(seed, update, off + 1, T, 1, F)[:, 0], m[:, 1])
    assert np.array_equal(D.dropout_multiplier(seed, update + (1 << 32), off, T, B, F), m)
    # F is a prefix: the first 123 features of a 300-wide batch are the 123-wide batch
    assert np.array_equal(D.dropout_multiplier(seed, update, off, T, B, 123), m[:, :, :123])


def test_dropout_multiplier_is_bernoulli_half_and_independent_across_positions():
    m = D.dropout_multiplier(1, 0, 0, 200, 16, 256)
    n = m.size
    kept = float((m > 0).mean())
    assert abs(kept - 0.5) < 5 * 0.5 / np.sqrt(n)
    for a, b in [(m[:, :, :-1], m[:, :, 1:]), (m[:-1], m[1:]), (m[:, :-1], m[:, 1:])]:
        assert abs(np.corrcoef(a.ravel(), b.ravel())[0, 1]) < 6 / np.sqrt(n)


def test_box_muller_u_is_the_float32_rounding_of_the_top_24_bits_plus_a_half():
    x = np.array([0, 0xff, 0x100, (1 << 31) - 1, 1 << 31, 0x80000100, 0xfffffeff, 0xffffffff], dtype=np.uint64)
    u = D.uniform_u(x)
    top = (x >> np.uint64(8)).astype(np.float64)
    # below 2^23 the half fits; above it the sum rounds to even
    small = top < 2 ** 23
    assert np.array_equal(u[small], (top[small] + 0.5) / 2 ** 24)
    assert np.array_equal(u[~small] * 2 ** 24, np.where(top[~small] % 2 == 0, top[~small], top[~small] + 1))
    assert u.min() > 0 and u.max() == 1.0
    e0, e1, r = D.box_muller(np.array([0xffffffff], np.uint64), np.array([0], np.uint64))
    assert r[0] == 0.0 and e0[0] == 0.0 and e1[0] == 0.0
    assert np.array_equal(D.uniform_v(np.array([0xffffffff], np.uint64)), [1.0 - 2.0 ** -24])


def test_eps_groups_follow_the_counter_and_the_pairing():
    seed, update, q = 0x123456789abcdef0, (3 << 32) | 9, np.array([0, 5, (1 << 33) + 1], dtype=np.uint64)
    eps, rad = D.eps_groups(seed, update, q, D.TAG_WEIGHT_NOISE)
    for i, qi in enumerate(q.tolist()):
        x, y, z, w = D.philox4x32_10(qi & 0xffffffff, qi >> 32, 9, 3 ^ D.TAG_WEIGHT_NOISE, seed & 0xffffffff, seed >> 32)
        ra, rb = np.sqrt(-2 * np.log(D.uniform_u(x))), np.sqrt(-2 * np.log(D.uniform_u(z)))
        va, vb = D.uniform_v(y), D.uniform_v(w)
        want = [ra * np.cos(2 * np.pi * va), ra * np.sin(2 * np.pi * va), rb * np.cos(2 * np.pi * vb),
                rb * np.sin(2 * np.pi * vb)]
        assert np.allclose(eps[i], want, rtol=0, atol=1e-15) and np.allclose(rad[i], [ra, ra, rb, rb], rtol=0, atol=0)


def test_eps_is_standard_normal():
    from scipy import stats
    eps, _ = D.eps_groups(1, 0, np.arange(50000, dtype=np.uint64), D.TAG_ADAPTIVE)
    e = eps.ravel()
    assert stats.kstest(e, "norm").pvalue > 1e-4
    assert abs(np.corrcoef(e[:-1], e[1:])[0, 1]) < 5 / np.sqrt(e.size)


def _shapes():
    return [("conv", O.param_shapes(O.make_config(num_features=123, dims_bidir=[128, 128], subsample=[1, 2]))),
            ("content", CO.param_shapes(CO.make_config(num_features=40, dims_bidir=[256], subsample=[1])))]


@pytest.mark.parametrize("name,shapes", _shapes(), ids=[s[0] for s in _shapes()])
def test_flat_layout_starts_each_parameter_at_a_multiple_of_64_and_groups_never_straddle(name, shapes):
    counts = [int(np.prod(s)) for s in shapes.values()]
    spans, n = D.flat_layout(counts)
    assert any(c % 4 for c in counts) or name == "content"
    for (o, c), (o2, _) in zip(spans, spans[1:] + [(n, 0)]):
        assert o % D.PARAM_ALIGN == 0 and o + c <= o2 < o + c + D.PARAM_ALIGN
        # so the first group of four starts at the parameter, and the last one ends in the padding, never in the next
        assert (o + c + 3) // 4 * 4 <= o2
    # eps of the padding is zero, and a parameter of count % 4 != 0 keeps only its own elements
    subject = [RO.is_noise_subject(k) for k in shapes]
    eps, rad = D.weight_noise_eps(3, 0, spans, n, subject)
    inside = np.zeros(n, bool)
    for o, c in spans:
        inside[o:o + c] = True
    assert not eps[~inside].any() and not rad[~inside].any()
    for (k, (o, c)), s in zip(zip(shapes, spans), subject):
        assert eps[o:o + c].any() == s, k


@pytest.mark.parametrize("name,shapes", _shapes(), ids=[s[0] for s in _shapes()])
def test_the_attention_parameters_are_not_noise_subjects_and_everything_else_is(name, shapes):
    att = [k for k in shapes if not RO.is_noise_subject(k)]
    assert att and all("/generator/att_trans/" in k and k.split("/")[4] in ("conv_att", "cont_att") for k in att)
    assert all(RO.is_noise_subject(k) for k in shapes if "/att_trans/conv_att/" not in k and "/att_trans/cont_att/" not in k)


def test_the_three_streams_never_share_a_counter():
    """Dropout keys its fourth counter word with 0xD0 << 24 | f / 128, weight noise with update_hi ^ 0x57 << 24,
    adaptive noise with update_hi: for updates below 2^56 and F below 2^31 the top byte of that word tells the three
    apart (0xD0, 0x57, 0), whatever the first three words."""
    updates = [0, 1, (1 << 31) + 5, (1 << 32) + 3, (1 << 56) - 1]
    adaptive = {((u >> 32) ^ D.TAG_ADAPTIVE) >> 24 for u in updates}
    weight = {((u >> 32) ^ D.TAG_WEIGHT_NOISE) >> 24 for u in updates}
    dropout = {(D.TAG_DROPOUT | (f >> 7)) >> 24 for f in [0, 127, 128, 1000, (1 << 31) - 1]}
    assert adaptive == {0} and weight == {0x57} and dropout == {0xD0}
    # and the draws differ: the same seed, update and group under the two noise tags
    a, _ = D.eps_groups(9, 0, np.arange(1000, dtype=np.uint64), D.TAG_ADAPTIVE)
    w, _ = D.eps_groups(9, 0, np.arange(1000, dtype=np.uint64), D.TAG_WEIGHT_NOISE)
    assert abs(np.corrcoef(a.ravel(), w.ravel())[0, 1]) < 5 / np.sqrt(a.size)
