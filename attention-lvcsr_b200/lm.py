"""FST language model for shallow fusion: the reader of OpenFST's binary ``vector`` format and the arc table the
library takes (lvsr_model_set_lm, include/lvsr_b200.h).

The reference loads the FST with PyFST (lvsr/ops.py:36-47) and maps the network's characters to the FST's input
symbols through ``character_map`` (lvsr/bricks/language_models.py:99-117).  Here the file is read directly.  Only
what a ``standard`` or ``log`` vector FST with an embedded input symbol table contains is accepted; anything else is
refused with a ValueError.  The format is implemented from its definition (header, symbol tables, per-state final
weight and arcs); it has not been checked against a file written by OpenFST itself.
"""
import struct

import numpy as np

FST_MAGIC = 2125659606
SYMBOL_TABLE_MAGIC = 2125658996
HAS_ISYMBOLS = 1
HAS_OSYMBOLS = 2
ARC_TYPES = ("standard", "log")
ARC_DTYPE = np.dtype([("ilabel", "<i4"), ("olabel", "<i4"), ("weight", "<f4"), ("nextstate", "<i4")])


class _Reader(object):
    def __init__(self, data, path):
        self.data, self.pos, self.path = data, 0, path

    def take(self, n):
        if self.pos + n > len(self.data):
            raise ValueError("%s: truncated FST file" % self.path)
        b = self.data[self.pos:self.pos + n]
        self.pos += n
        return b

    def unpack(self, fmt):
        return struct.unpack("<" + fmt, self.take(struct.calcsize("<" + fmt)))

    def string(self):
        (n,) = self.unpack("i")
        if n < 0:
            raise ValueError("%s: bad string length %d" % (self.path, n))
        return self.take(n).decode("utf-8")

    def symbols(self):
        (magic,) = self.unpack("i")
        if magic != SYMBOL_TABLE_MAGIC:
            raise ValueError("%s: bad symbol table magic %d" % (self.path, magic))
        self.string()
        _available, size = self.unpack("qq")
        table = {}
        for _ in range(size):
            sym = self.string()
            (key,) = self.unpack("q")
            table[sym] = key
        return table


def read_fst(path):
    """OpenFST binary vector FST -> dict(start, num_states, isyms {symbol: code}, arcs: per state a structured array
    of (ilabel, olabel, weight, nextstate)).  Weights are float32 costs, as OpenFST stores them."""
    with open(path, "rb") as f:
        r = _Reader(f.read(), path)
    (magic,) = r.unpack("i")
    if magic != FST_MAGIC:
        raise ValueError("%s: not an OpenFST binary file (magic %d)" % (path, magic))
    fst_type, arc_type = r.string(), r.string()
    if fst_type != "vector":
        raise ValueError("%s: FST type %r is not supported (only 'vector')" % (path, fst_type))
    if arc_type not in ARC_TYPES:
        raise ValueError("%s: arc type %r is not supported (only 'standard' and 'log')" % (path, arc_type))
    _version, flags, _properties, start, num_states, _num_arcs = r.unpack("iiQqqq")
    if not flags & HAS_ISYMBOLS:
        raise ValueError("%s: the FST has no input symbol table, which the character map needs" % path)
    isyms = r.symbols()
    if flags & HAS_OSYMBOLS:
        r.symbols()
    if not 0 <= start < num_states:
        raise ValueError("%s: start state %d outside [0, %d)" % (path, start, num_states))
    arcs = []
    for _ in range(num_states):
        _final, narcs = r.unpack("fq")
        if narcs < 0:
            raise ValueError("%s: bad arc count %d" % (path, narcs))
        a = np.frombuffer(r.take(narcs * ARC_DTYPE.itemsize), dtype=ARC_DTYPE)
        if narcs and (a["nextstate"].min() < 0 or a["nextstate"].max() >= num_states):
            raise ValueError("%s: an arc leads outside the %d states" % (path, num_states))
        arcs.append(a)
    return dict(start=int(start), num_states=int(num_states), isyms=isyms, arcs=arcs)


def remap_table(isyms, character_map):
    """remap[nn label] = FST input label through the characters (lvsr/bricks/language_models.py:107-113)."""
    fst_chars = dict(isyms)
    fst_chars.pop("<eps>", None)
    if len(fst_chars) != len(character_map):
        raise ValueError("the FST has %d input symbols besides <eps>, the character map %d characters"
                         % (len(fst_chars), len(character_map)))
    try:
        return {int(character_map[ch]): int(code) for ch, code in fst_chars.items()}
    except KeyError as e:
        raise ValueError("FST input symbol %s is not in the character map" % e)


def arc_table(fst, remap, num_phonemes):
    """CSR arc table in NN label space for lvsr_model_set_lm: (offsets int64 [S+1], label int32 = nn label + 1 with
    0 = epsilon, next int32, weight float32), each state's arcs sorted by (label, next state).  Arcs whose input
    label is no character can never be taken and are left out."""
    if sorted(remap) != list(range(num_phonemes)):
        raise ValueError("the character map must cover the labels 0..%d exactly" % (num_phonemes - 1))
    codes = list(remap.values())
    if len(set(codes)) != len(codes) or 0 in codes:
        raise ValueError("the FST input symbols of the characters must be distinct and not epsilon")
    lut = np.full(max(codes) + 1, -1, dtype=np.int32)
    lut[0] = 0
    for nn, code in remap.items():
        lut[code] = nn + 1
    offsets = np.zeros(fst["num_states"] + 1, dtype=np.int64)
    labels, nexts, weights = [], [], []
    for s, a in enumerate(fst["arcs"]):
        il = a["ilabel"].astype(np.int64)
        lab = np.where((il >= 0) & (il < len(lut)), lut[np.clip(il, 0, len(lut) - 1)], -1).astype(np.int32)
        keep = lab >= 0
        lab, nxt, w = lab[keep], a["nextstate"][keep].astype(np.int32), a["weight"][keep].astype(np.float32)
        order = np.lexsort((nxt, lab))
        labels.append(lab[order])
        nexts.append(nxt[order])
        weights.append(w[order])
        offsets[s + 1] = offsets[s] + len(order)
    cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs) if xs else np.zeros(0, dt), dtype=dt)
    return dict(start=fst["start"], num_states=fst["num_states"], offsets=offsets, label=cat(labels, np.int32),
                next=cat(nexts, np.int32), weight=cat(weights, np.float32))


def load(path, character_map, num_phonemes):
    """read_fst + remap_table + arc_table."""
    fst = read_fst(path)
    return arc_table(fst, remap_table(fst["isyms"], character_map), num_phonemes)
