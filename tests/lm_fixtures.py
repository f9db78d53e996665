"""Seeded FSTs that reach the edges of the LM kernels (csrc/lm.cu), for tests/test_gpu_lm_matrix.py and the CPU file
that pins their properties (tests/test_lm_matrix_cpu.py).  Everything is in NN label space (label = symbol + 1,
0 = epsilon) as lists or arrays of (label, next, weight) per state, and written as an OpenFST vector file whose input
symbol 'c<k>' has code k + 1, so the identity character map {'c<k>': k} maps it back."""
import importlib.util
import os
import struct

import numpy as np

import lm_oracle as LO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bench_lm_search():
    spec = importlib.util.spec_from_file_location("bench_lm_search", os.path.join(ROOT, "tools", "bench_lm_search.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _arrays(a):
    if isinstance(a, tuple):
        return [np.asarray(x) for x in a]
    lab = np.array([t[0] for t in a], dtype=np.int32)
    nxt = np.array([t[1] for t in a], dtype=np.int32)
    return lab, nxt, np.array([t[2] for t in a], dtype=np.float32)


def write(path, V, num_states, start, arcs, arc_type="standard"):
    """arcs[s] = [(label, next, weight)] or (labels, nexts, weights) arrays -> OpenFST vector file; returns the
    character map."""
    dt = np.dtype([("ilabel", "<i4"), ("olabel", "<i4"), ("weight", "<f4"), ("nextstate", "<i4")])
    s = lambda t: struct.pack("<i", len(t)) + t.encode()
    syms = [("<eps>", 0)] + [("c%d" % k, k + 1) for k in range(V)]
    narcs = sum(len(_arrays(a)[0]) for a in arcs)
    parts = [struct.pack("<i", 2125659606), s("vector"), s(arc_type),
             struct.pack("<iiQqqq", 2, 1, 0, start, num_states, narcs),
             struct.pack("<i", 2125658996), s("chars"), struct.pack("<qq", V + 1, len(syms))]
    parts += [s(k) + struct.pack("<q", v) for k, v in syms]
    for a in arcs:
        lab, nxt, wt = _arrays(a)
        rec = np.zeros(len(lab), dtype=dt)
        rec["ilabel"], rec["olabel"], rec["weight"], rec["nextstate"] = lab, lab, wt, nxt
        parts.append(struct.pack("<fq", 0.0, len(rec)) + rec.tobytes())
    with open(path, "wb") as f:
        f.write(b"".join(parts))
    return {"c%d" % k: k for k in range(V)}


def ngram(V, seed):
    """LO.char_ngram at vocabulary V, with n_tri capped below V * V (the generator draws distinct histories and would
    loop forever beyond it)."""
    n_tri = min(60, V * V - 1)
    return LO.char_ngram(V, seed=seed, n_tri=n_tri, dup=min(6, n_tri), dead=2)


# ---- set sizes and closure caps ---------------------------------------------------------------------------------

CLOSURE_OK, CLOSURE_OVER = 32, 33


def limits_fst(V, seed):
    """Start 0.  Symbol n - 1 (n = 1..8) leads to a set of exactly n states: half of them by the transition, the rest
    over an epsilon chain from its first target.  Symbol 8 leads to gateway P, whose symbol 0 leads to a state with an
    epsilon closure of exactly CLOSURE_OK states; symbol 9 to gateway Q, whose symbol 0 leads to one of CLOSURE_OVER.
    Every other state has arcs on a few symbols back into the sets, so each set's cost row has finite entries.
    Returns (num_states, start, arcs, info) with info: sets {n: symbol}, P, Q."""
    assert V >= 10
    rng = np.random.RandomState(seed)
    w = lambda: float(np.float32(rng.uniform(-1.0, 3.0)))
    arcs = [[]]
    add = lambda: arcs.append([]) or len(arcs) - 1
    targets = {}
    for n in range(1, 9):
        states = [add() for _ in range(n)]
        direct = (n + 1) // 2
        for s in states[:direct]:
            arcs[0].append((n, s, w()))
        for a, b in zip([states[0]] + states[direct:-1], states[direct:]):
            arcs[a].append((0, b, w()))
        targets[n] = states
    P, Q = add(), add()
    arcs[0] += [(9, P, w()), (10, Q, w())]

    def closure(size):
        """a DAG of `size` states: a binary tree from its root plus cross arcs to later states (diamonds)"""
        xs = [add() for _ in range(size)]
        for i, x in enumerate(xs):
            for j in (2 * i + 1, 2 * i + 2):
                if j < size:
                    arcs[x].append((0, xs[j], w()))
            if i + 3 < size and i % 3 == 0:
                arcs[x].append((0, xs[i + 3], w()))
        return xs

    ok, over = closure(CLOSURE_OK), closure(CLOSURE_OVER)
    arcs[P].append((1, ok[0], w()))
    arcs[Q].append((1, over[0], w()))
    inner = [s for n in range(1, 8) for s in targets[n]]
    for s in inner + ok:
        for c in rng.choice(V, size=3, replace=False):
            arcs[s].append((int(c) + 1, int(rng.choice(inner[:6])), w()))
    arcs = [sorted(a) for a in arcs]
    return len(arcs), 0, arcs, dict(sets={n: n - 1 for n in range(1, 9)}, P=P, Q=Q)


# ---- closure order ----------------------------------------------------------------------------------------------

GROUP = 7


def order_fst(V, seed, groups=24):
    """Epsilon closures whose discovery order is not a topological order.  States come in groups of GROUP; epsilon
    arcs only go from a higher to a lower state of the same group (so every closure stays in one group and holds at
    most 7 states, and there is no cycle): a chain 6 deep from the group's top state, parallel arcs between the same
    two states, and random diamonds.  Every arc labelled c leads into 1-3 states of c's group, so the transition's
    set often holds a state the epsilon arcs also reach (and, sorted by state, before the state they come from).
    Weights are mixed-sign, as in a weight-pushed FST.  State 0 is the start; it has no epsilon arcs."""
    rng = np.random.RandomState(seed)
    w = lambda: float(np.float32(rng.uniform(-2.0, 3.0)))
    S = 1 + groups * GROUP
    arcs = [[] for _ in range(S)]
    base = lambda g: 1 + g * GROUP
    label_group = rng.randint(groups, size=V)
    for g in range(groups):
        b = base(g)
        for i in range(GROUP - 1, 0, -1):
            arcs[b + i].append((0, b + i - 1, w()))
        for _ in range(int(rng.randint(2, 6))):
            i = int(rng.randint(2, GROUP))
            j = int(rng.randint(0, i - 1))
            arcs[b + i].append((0, b + j, w()))
        i = int(rng.randint(1, GROUP))
        arcs[b + i].append((0, b + i - 1, w()))              # parallel to the chain's arc
    for s in range(S):
        for c in rng.choice(V, size=max(1, V // 2), replace=False):
            g = int(label_group[c])
            for t in rng.choice(GROUP, size=int(rng.randint(1, 4)), replace=False):
                arcs[s].append((int(c) + 1, base(g) + int(t), w()))
    return S, 0, [sorted(a) for a in arcs]


# ---- the benchmark's 4-gram and its variants --------------------------------------------------------------------

def four_gram(seed=5):
    """tools/bench_lm_search.py's synthetic character 4-gram over 32 symbols (33,825 states, 1,116,224 arcs), start 0:
    (V, num_states, start, arcs[s] = (labels, nexts, weights))."""
    b = _bench_lm_search()
    S, arcs = b.four_gram(seed)
    return b.V, S, 0, arcs


LONG_WALK = dict(rows=6, steps=320, seed=8)       # the long walks on the 4-gram: set weights reach the hundreds


def uniform_walk(V, rows, steps, seed):
    """[steps, rows] symbols drawn uniformly from a seeded stream (every symbol of the 4-gram leads somewhere)."""
    return np.random.RandomState(seed).randint(V, size=(steps, rows))


def pushed(num_states, arcs, seed, spread=3.0):
    """Every arc s -> t reweighted by w + phi(s) - phi(t) with a seeded potential phi in [-spread, spread]: the path
    weights change by the end points only, as weight pushing changes them, and many arcs become negative."""
    phi = np.random.RandomState(seed).uniform(-spread, spread, size=num_states)
    return [(lab, nxt, (w.astype(np.float64) + phi[s] - phi[nxt]).astype(np.float32)) for s, (lab, nxt, w) in enumerate(arcs)]


def wide(V, num_states, arcs, seed, parallel=(9, 14)):
    """A non-deterministic start state W added to `arcs` (a 4-gram): on every symbol it leads to 2-4 distinct
    unigram-history states, each over a run of `parallel` arcs with the same label and next state, so the state holds
    more than 1,000 arcs and the first arc of a label's run is one of many equal labels.  With 4 targets the set three
    symbols later holds exactly 7 states (the targets' trigram histories, then one each of history 2, 1 and 0).
    Returns (num_states + 1, W, arcs)."""
    rng = np.random.RandomState(seed)
    labs, nxts, ws = [], [], []
    for c in range(V):
        k = 4 if c % 4 == 0 else int(rng.randint(2, 5))
        for t in sorted(rng.choice(V, size=k, replace=False)):
            n = int(rng.randint(*parallel))
            labs += [c + 1] * n
            nxts += [1 + int(t)] * n
            ws += list(rng.uniform(0.5, 4.0, size=n))
    W = num_states
    return num_states + 1, W, list(arcs) + [(np.array(labs, np.int32), np.array(nxts, np.int32), np.array(ws, np.float32))]


def memo(fst):
    """MemoFST of an LO.FST (LO.from_tables of what the library received)."""
    return MemoFST(fst.num_states, fst.start, fst.arcs)


def oracle_fst(num_states, start, arcs):
    """The oracle's FST of an arc list, for checks that need no library."""
    return MemoFST(num_states, start, [list(zip(*[x.tolist() for x in _arrays(a)])) for a in arcs])


_costs_row = LO.costs_row


def memo_rows(fst, states, V, no_transition_cost):
    """LO.costs_row through the memo of a MemoFST (what a test patches LO.costs_row with, so that LO.lm_path,
    LO.next_state and LO.computers share it)."""
    return fst.row(states, V, no_transition_cost) if isinstance(fst, MemoFST) else _costs_row(fst, states, V, no_transition_cost)


class MemoFST(LO.FST):
    """LO.FST whose advance and cost rows are memoised by frozen set: walks over many rows and the hypotheses of a
    search revisit the same sets."""

    def __init__(self, num_states, start, arcs):
        super(MemoFST, self).__init__(num_states, start, arcs)
        self._adv, self._rows = {}, {}

    def advance(self, states, character):
        key = (frozenset(states.items()), character)
        if key not in self._adv:
            self._adv[key] = super(MemoFST, self).advance(states, character)
        return dict(self._adv[key])

    def row(self, states, V, no_transition_cost):
        key = (frozenset(states.items()), V, no_transition_cost)
        if key not in self._rows:
            self._rows[key] = _costs_row(self, states, V, no_transition_cost)
        return self._rows[key]
