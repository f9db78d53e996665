"""The FST generators of tests/lm_fixtures.py reach what tests/test_gpu_lm_matrix.py claims they reach: sets of 1 to
7 states and the refused 8, epsilon closures of 32 and 33 states, closures whose discovery order is not a
topological order, runs of equal labels behind one state of more than 1,000 arcs, mixed-sign weights, and walks of at
least 300 symbols whose float32 restatement misses the cost bound the GPU is held to."""
import math
from collections import deque

import numpy as np
import pytest

import lm_fixtures as F
import lm_oracle as LO

NTC = 20.0


def _walk(fst, V, steps, seed):
    """Sets and cost rows of one seeded walk (symbols the set knows, 9 times in 10)."""
    rng = np.random.RandomState(seed)
    s, row = LO.initial(fst, V, NTC)
    out = [(s, row)]
    for _ in range(steps):
        known = np.flatnonzero(row < np.float32(NTC))
        y = int(rng.choice(known)) if known.size and rng.rand() < 0.9 else int(rng.randint(V))
        s, row = LO.next_state(fst, s, y, V, NTC)
        out.append((s, row))
    return out


@pytest.mark.parametrize("V", [2, 31, 33, 63, 64, 65, 127, 128])
def test_ngram_builds_at_every_width(V):
    S, start, arcs = F.ngram(V, seed=7)
    labels = {lab for a in arcs for lab, _, _ in a}
    assert labels <= set(range(V + 1)) and max(labels) >= V - (V > 2)      # symbols past 32 carry arcs
    fst = LO.FST(S, start, arcs)
    sizes = [len(s) for seed in range(6) for s, _ in _walk(fst, V, 12, seed)]
    assert max(sizes) >= 2


def test_limits_fst_reaches_every_set_size_and_both_closure_caps():
    V = 32
    S, start, arcs, info = F.limits_fst(V, seed=3)
    fst = LO.FST(S, start, arcs)
    s0, row0 = LO.initial(fst, V, NTC)
    assert s0 == {0: 0.0} and np.isfinite(row0).all()
    for n, y in info["sets"].items():
        assert len(fst.advance(s0, y + 1)) == n
        if n <= 7:
            s, row = LO.next_state(fst, s0, y, V, NTC)
            assert len(s) == n and (row < NTC).sum() >= 1          # each set's row has a finite cost
        else:
            with pytest.raises(ValueError, match="more than 7"):
                LO.next_state(fst, s0, y, V, NTC)
    P, _ = LO.next_state(fst, s0, 8, V, NTC)
    Q, _ = LO.next_state(fst, s0, 9, V, NTC)
    assert set(P) == {info["P"]} and set(Q) == {info["Q"]}
    assert len(fst.advance(P, 1)) == F.CLOSURE_OK and len(fst.advance(Q, 1)) == F.CLOSURE_OVER
    assert LO.costs_row(fst, P, V, NTC)[0] < NTC
    assert any(w < 0 for a in arcs for _, _, w in a)


def _discovery_expand(fst, states):
    """expand with the closure's weights propagated in discovery order (each state once, in the order the search
    found it) instead of a topological order: what a kernel without Kahn's ordering computes."""
    order, seen, queue = [], set(states), deque(states)
    while queue:
        q = queue.popleft()
        order.append(q)
        for _, nxt, _, _ in fst.get_arcs(q, LO.EPSILON):
            if nxt not in seen:
                seen.add(nxt)
                queue.append(nxt)
    out = dict(states)
    for q in order:
        for _, nxt, _, w in fst.get_arcs(q, LO.EPSILON):
            out[nxt] = fst.combine_weights(out.get(nxt), out[q] + w)
    return out


def _closure_shapes(fst):
    """(parallel epsilon arcs, states with 2 or more epsilon predecessors, longest epsilon chain)"""
    parallel, preds, depth = 0, {}, {}
    for s, a in enumerate(fst.arcs):
        eps = [n for lab, n, _ in a if lab == 0]
        parallel += len(eps) - len(set(eps))
        for n in set(eps):
            preds[n] = preds.get(n, 0) + 1

    def d(s):
        if s not in depth:
            depth[s] = 1 + max([d(n) for lab, n, _ in fst.arcs[s] if lab == 0], default=0)
        return depth[s]
    return parallel, sum(1 for v in preds.values() if v >= 2), max(d(s) for s in range(fst.num_states)) - 1


def test_order_fst_closures_need_a_topological_order():
    V = 32
    S, start, arcs = F.order_fst(V, seed=11)
    fst = LO.FST(S, start, arcs)
    parallel, diamonds, chain = _closure_shapes(fst)
    assert parallel > 0 and diamonds > 0 and chain >= 6
    assert any(w < 0 for a in arcs for _, _, w in a) and any(w > 0 for a in arcs for _, _, w in a)
    wrong = into_own = sizes = 0
    for seed in range(8):
        prev = None
        for s, _ in _walk(fst, V, 16, seed):
            sizes = max(sizes, len(s))
            if prev is not None:
                for c in range(1, V + 1):
                    t = fst.transition(prev, c)
                    if not t:
                        continue
                    into_own += any(n in t for q in t for _, n, _, _ in fst.get_arcs(q, LO.EPSILON))
                    good, bad = fst.expand(t), _discovery_expand(fst, t)
                    wrong += any(abs(good[k] - bad[k]) > 1e-6 for k in good)
            prev = s
    print("closures the discovery order gets wrong:", wrong, "transitions into their own closure:", into_own)
    assert wrong > 10 and into_own > 10 and sizes == 7


def test_four_gram_walks_reach_hundreds_and_float32_misses_the_bound():
    """The long walks of the GPU file (F.LONG_WALK, on the 4-gram and its pushed variant) restated with float32
    weights and log-adds: their cost rows break the bound the GPU rows are held to (rtol = atol = 1e-5)."""
    V, S, start, arcs = F.four_gram()
    assert S == 33825 and sum(len(a[0]) for a in arcs) == 1116224
    W = F.LONG_WALK
    assert W["steps"] >= 300
    ys = F.uniform_walk(V, **W)
    push = F.pushed(S, arcs, seed=1)
    assert (np.concatenate([a[2] for a in push]) < 0).mean() > 0.1
    for a in (arcs, push):
        fst = F.oracle_fst(S, start, a)
        f32 = _F32(S, start, fst.arcs)
        s0, _ = LO.initial(fst, V, NTC)
        sets, sets32 = [s0] * W["rows"], [LO.initial(f32, V, NTC)[0]] * W["rows"]
        over, heaviest = 0.0, 0.0
        for step in ys:
            for r, y in enumerate(step):
                sets[r], row = LO.next_state(fst, sets[r], int(y), V, NTC)
                sets32[r], row32 = LO.next_state(f32, sets32[r], int(y), V, NTC)
                want = row.astype(np.float64)
                over = max(over, float((np.abs(row32.astype(np.float64) - want) - 1e-5 * (1 + np.abs(want))).max()))
                heaviest = max(heaviest, max(sets[r].values()))
        print("set weights up to %.1f; the float32 restatement exceeds the row bound by %.2e" % (heaviest, over))
        assert heaviest > 300 and over > 0


class _F32(LO.FST):
    """The FST operations with every weight and log-add rounded to float32."""

    @staticmethod
    def combine_weights(*args):
        xs = [np.float32(x) for x in args if x is not None]
        m = max(xs)
        return np.float32(m - np.float32(np.log(np.sum(np.exp(np.array([m - x for x in xs], np.float32))))))


def test_wide_state_has_runs_of_equal_labels_and_reaches_seven_states():
    V, S, start, arcs = F.four_gram()
    S2, W, arcs2 = F.wide(V, S, arcs, seed=3)
    lab, nxt, w = arcs2[W]
    assert len(lab) > 1000 and W == S and S2 == S + 1
    for c in range(1, V + 1):
        targets, counts = np.unique(nxt[lab == c], return_counts=True)
        assert 2 <= len(targets) <= 4 and counts.min() >= 2
    fst = F.oracle_fst(S2, W, arcs2)
    # a lower_bound that stops at any arc of the label (here: the middle of the run) loses targets or weights
    s0 = fst.expand({W: 0.0})
    lost = 0
    for c in range(1, V + 1):
        full = fst.transition(s0, c)
        run = [a for a in fst.arcs[W] if a[0] == c]
        part = {}
        for _, n, wt in run[len(run) // 2:]:
            part[n] = fst.combine_weights(part.get(n), wt)
        lost += set(part) != set(full) or any(abs(part[k] - full[k]) > 1e-6 for k in part)
    assert lost == V
    sizes = [len(s) for s, _ in _walk(fst, V, 6, 1)]
    rng = np.random.RandomState(2)
    s = fst.expand({W: 0.0})
    for y in [0] + list(rng.randint(V, size=4)):                 # symbol 0 leads to 4 targets
        s = fst.advance(s, int(y) + 1)
        sizes.append(len(s))
    assert max(sizes) == 7 and min(sizes[1:]) >= 3


def test_fast_writer_round_trips_through_the_reader(tmp_path):
    from helpers import package
    S, start, arcs = F.order_fst(5, seed=2, groups=3)
    for arc_type in ("standard", "log"):
        path = str(tmp_path / ("o_%s.fst" % arc_type))
        cmap = F.write(path, 5, S, start, arcs, arc_type=arc_type)
        got = LO.from_tables(package().lm.load(path, cmap, 5))
        assert got.start == start and got.num_states == S
        for s in range(S):
            assert sorted(got.arcs[s]) == sorted((l, n, float(np.float32(w))) for l, n, w in arcs[s])
    assert math.isfinite(F.MemoFST(S, start, got.arcs).row({start: 0.0}, 5, NTC)[0])
