"""Float64 numpy restatement of the reference's FST language model and shallow fusion, the checker of the LM kernels:
FST.transition / expand / combine_weights (lvsr/ops.py:36-110, the `max` form of combine_weights), FSTCostsOp,
FSTTransitionOp (:113-233), ShallowFusionReadout and LMEmitter (lvsr/bricks/language_models.py).  Also a writer of
OpenFST's binary vector format and a seeded character n-gram FST with backoff, for tests and benchmarks."""
import math
import struct
from collections import OrderedDict, defaultdict, deque

import numpy as np

from oracle import lvsr_oracle as O

EPSILON = 0
MAX_STATES = 7
NOT_STATE = -1


class CycleError(Exception):
    pass


class FST(object):
    """In NN label space: arcs[s] = [(label, next, weight)], label = nn symbol + 1, 0 = epsilon (the remap of the
    reference applied to the arcs instead of the queries)."""

    def __init__(self, num_states, start, arcs):
        self.num_states, self.start, self.arcs = num_states, start, arcs

    @staticmethod
    def combine_weights(*args):
        m = max(x for x in args if x is not None)       # Python 2's max, where None orders below every number
        return m - math.log(sum(math.exp(m - x) for x in args if x is not None))

    def get_arcs(self, state, character):
        return [(state, nxt, lab, float(w)) for lab, nxt, w in self.arcs[state] if lab == character]

    def transition(self, states, character):
        arcs = [a for s in states for a in self.get_arcs(s, character)]
        next_states = {}
        for next_state in {a[1] for a in arcs}:
            next_states[next_state] = self.combine_weights(*[states[a[0]] + a[3] for a in arcs if a[1] == next_state])
        return next_states

    def expand(self, states):
        seen = set(states)
        depends = defaultdict(list)
        queue = deque(states)
        while queue:
            state = queue.popleft()
            for arc in self.get_arcs(state, EPSILON):
                depends[arc[1]].append((arc[0], arc[3]))
                if arc[1] in seen:
                    continue
                queue.append(arc[1])
                seen.add(arc[1])
        order = _toposort({k: {s for s, _ in v} for k, v in depends.items()})
        next_states = dict(states)
        for next_state in order:
            next_states[next_state] = self.combine_weights(
                *([next_states.get(next_state)] + [next_states[p] + w for p, w in depends[next_state]]))
        return next_states

    def advance(self, states, character):
        return self.expand(self.transition(states, character))


def _toposort(deps):
    """toposort_flatten for the closure graph; a cycle (a self-loop included) raises CycleError."""
    nodes = set(deps) | {d for v in deps.values() for d in v}
    indeg = {n: len(deps.get(n, ())) for n in nodes}
    users = defaultdict(list)
    for n, ds in deps.items():
        for d in ds:
            users[d].append(n)
    ready = sorted(n for n in nodes if indeg[n] == 0)
    order = []
    while ready:
        n = ready.pop(0)
        order.append(n)
        for u in users[n]:
            indeg[u] -= 1
            if indeg[u] == 0:
                ready.append(u)
    if len(order) != len(nodes):
        raise CycleError()
    return order


def costs_row(fst, states, V, no_transition_cost):
    """FSTCostsOp for one set: float32 row of V costs."""
    costs = np.ones(V, dtype=np.float32) * np.float32(no_transition_cost)
    if states:
        total = fst.combine_weights(*states.values())
        for c in range(V):
            nxt = fst.advance(states, c + 1)
            if nxt:
                costs[c] = fst.combine_weights(*nxt.values()) - total
    return costs


def initial(fst, V, no_transition_cost):
    s = fst.expand({fst.start: 0.0})
    return s, costs_row(fst, s, V, no_transition_cost)


def next_state(fst, states, y, V, no_transition_cost):
    """FSTTransitionOp + FSTCostsOp for one row; a set over MAX_STATES raises (numpy.pad with a negative width)."""
    s = fst.advance(states, int(y) + 1)
    if len(s) > MAX_STATES:
        raise ValueError("more than %d states" % MAX_STATES)
    return s, costs_row(fst, s, V, no_transition_cost)


def log_softmax(x):
    return O.log_softmax(x)


def fused_costs(logits, add, o):
    """ShallowFusionReadout.readout then LMEmitter.costs: -x for every symbol."""
    x = o["am_beta"] * np.asarray(logits, dtype=np.float64)
    if o["normalize_am_weights"]:
        x = log_softmax(x)
    lm = -np.asarray(add, dtype=np.float64)
    if o["normalize_lm_weights"]:
        lm = log_softmax(lm)
    x = x + o["weight"] * lm
    if o["normalize_tot_weights"]:
        x = log_softmax(x)
    return -x


def lm_path(fst, labels, labels_mask, V, no_transition_cost):
    """LanguageModel.evaluate: add [L, B, V], the row in force before each label; masked steps keep the state."""
    L, B = labels.shape
    out = np.zeros((L, B, V), dtype=np.float32)
    for b in range(B):
        s, row = initial(fst, V, no_transition_cost)
        for i in range(L):
            if i > 0 and (labels_mask is None or labels_mask[i - 1, b]):
                s = fst.advance(s, int(labels[i - 1, b]) + 1)
                row = costs_row(fst, s, V, no_transition_cost)
            out[i, b] = row
    return out


def cost_matrix(cfg, params, fst, o, attended, attended_mask, labels, labels_mask=None, oracle=O):
    """generator.cost_matrix with the language model: LMEmitter.cost of the fused readout (`oracle`: the module of
    the attention's oracle, O or content_oracle)."""
    r = oracle.cost_matrix(cfg, params, attended, attended_mask, labels, labels_mask, return_all=True)
    logits = O.readout(cfg, params, r["states"], r["weighted_averages"])
    add = lm_path(fst, labels, labels_mask, cfg["num_phonemes"], o["no_transition_cost"])
    costs = np.take_along_axis(fused_costs(logits, add, o), labels[..., None], axis=-1)[..., 0]
    if labels_mask is not None:
        costs = costs * labels_mask
    return costs


def computers(cfg, params, fst, o):
    """initial / logprobs / next for O.beam_search with the LM state carried in the state dict (one entry per row:
    the set as a dict, and its cost row)."""
    V, ntc = cfg["num_phonemes"], o["no_transition_cost"]

    def f_init(att):
        st = O.initial_states(cfg, params, 1, att)
        s, row = initial(fst, V, ntc)
        st["lm_sets"] = np.array([s], dtype=object)
        st["lm_add"] = row[None, :]
        return st

    def f_logp(att, m, st):
        wa, _, _, _ = O.take_glimpses(cfg, params, att, None, m, st["weights"], st["step"], st["states"])
        return fused_costs(O.readout(cfg, params, st["states"], wa), st["lm_add"], o)

    def f_next(att, m, st, y):
        nxt = O.next_state_computer(cfg, params, att, m, OrderedDict((k, v) for k, v in st.items() if not k.startswith("lm_")), y)
        sets, rows = [], []
        for s, yy in zip(st["lm_sets"], y):
            s2, row = next_state(fst, s, yy, V, ntc)
            sets.append(s2)
            rows.append(row)
        out = np.empty(len(sets), dtype=object)
        out[:] = sets
        nxt["lm_sets"] = out
        nxt["lm_add"] = np.stack(rows) if rows else np.zeros((0, V), np.float32)
        return nxt

    return dict(initial=f_init, logprobs=f_logp, next=f_next)


# ---- OpenFST binary vector format (writer) --------------------------------------------------------------------
def _string(s):
    b = s.encode("utf-8")
    return struct.pack("<i", len(b)) + b


def _symbols(table):
    out = struct.pack("<i", 2125658996) + _string("syms") + struct.pack("<qq", max(table.values()) + 1, len(table))
    for sym, key in table.items():
        out += _string(sym) + struct.pack("<q", key)
    return out


def write_fst(path, num_states, start, arcs, isyms, osyms=None, magic=2125659606, fst_type="vector",
              arc_type="standard"):
    """arcs[s] = [(ilabel, olabel, weight, next)] in FST label space; isyms {symbol: code} or None."""
    flags = (1 if isyms is not None else 0) | (2 if osyms is not None else 0)
    narcs = sum(len(a) for a in arcs)
    out = struct.pack("<i", magic) + _string(fst_type) + _string(arc_type)
    out += struct.pack("<iiQqqq", 2, flags, 0, start, num_states, narcs)
    if isyms is not None:
        out += _symbols(isyms)
    if osyms is not None:
        out += _symbols(osyms)
    for s in range(num_states):
        out += struct.pack("<fq", 0.0, len(arcs[s]))
        for il, ol, w, nx in arcs[s]:
            out += struct.pack("<iifi", il, ol, w, nx)
    with open(path, "wb") as f:
        f.write(out)


def char_ngram(V, seed, n_tri=12, dup=3, dead=1):
    """Seeded character trigram FST with backoff in NN label space: state 0 = unigram, 1..V = bigram histories,
    then n_tri trigram histories, one start state without backoff (a symbol it has no arc for ends the
    hypothesis' LM) and `dead` dead ends (states without arcs) it leads to.  Trigram -> bigram -> unigram
    are epsilon chains two deep; `dup` bigram states get a second arc with the same label to a trigram state whose
    backoff is the first arc's target, so a closure revisits a state of the set it starts from.  Returns
    (num_states, start, arcs[s] = [(label, next, weight float32)])."""
    rng = np.random.RandomState(seed)
    w = lambda: float(np.float32(rng.uniform(0.1, 4.0)))
    big = lambda c: 1 + c
    tri_hist = []
    seen = set()
    while len(tri_hist) < n_tri:
        h = (int(rng.randint(V)), int(rng.randint(V)))
        if h not in seen:
            seen.add(h)
            tri_hist.append(h)
    tri = {h: 1 + V + i for i, h in enumerate(tri_hist)}
    start = 1 + V + n_tri
    dead_states = list(range(start + 1, start + 1 + dead))
    S = start + 1 + dead
    arcs = [[] for _ in range(S)]
    for c in range(V):                                   # unigram: every symbol
        arcs[0].append((c + 1, big(c), w()))
    for h in range(V):                                   # bigram: some symbols, backoff to unigram
        for c in rng.choice(V, size=max(1, V // 3), replace=False):
            c = int(c)
            arcs[big(h)].append((c + 1, tri.get((h, c), big(c)), w()))
        arcs[big(h)].append((0, 0, w()))
    for (h1, h2), s in tri.items():                      # trigram: some symbols, backoff to the bigram of h2
        for c in rng.choice(V, size=max(1, V // 4), replace=False):
            c = int(c)
            arcs[s].append((c + 1, tri.get((h2, c), big(c)), w()))
        arcs[s].append((0, big(h2), w()))
    for c in rng.choice(V, size=max(V // 2, 1), replace=False):   # start: some symbols, no backoff (others: dead)
        arcs[start].append((int(c) + 1, big(int(c)), w()))
    for (h1, h2), s in list(tri.items())[:dup]:          # duplicate label: bigram h1 --h2--> {bigram h2, trigram (h1,h2)}
        arcs[big(h1)].append((h2 + 1, big(h2), w()))
        arcs[big(h1)].append((h2 + 1, s, w()))
    for d in dead_states:                                # a symbol of the start state leads into a dead end
        arcs[start].append((int(rng.randint(V)) + 1, d, w()))
    return S, start, arcs


def to_file(path, V, num_states, start, arcs, seed=0):
    """Write an NN-space FST as an OpenFST file whose input symbols are a shuffled code assignment, and return the
    character_map that maps it back: character 'c<k>' is NN label k."""
    rng = np.random.RandomState(seed)
    codes = rng.permutation(V) + 1
    isyms = OrderedDict([("<eps>", 0)] + [("c%d" % k, int(codes[k])) for k in range(V)])
    fst_arcs = [[(0 if lab == 0 else int(codes[lab - 1]), 0, wt, nx) for lab, nx, wt in a] for a in arcs]
    write_fst(path, num_states, start, fst_arcs, isyms)
    return {"c%d" % k: k for k in range(V)}


def from_tables(t):
    """FST of lm.arc_table's output (what the library receives)."""
    arcs = []
    for s in range(t["num_states"]):
        a, b = t["offsets"][s], t["offsets"][s + 1]
        arcs.append([(int(l), int(n), float(w)) for l, n, w in zip(t["label"][a:b], t["next"][a:b], t["weight"][a:b])])
    return FST(t["num_states"], t["start"], arcs)
