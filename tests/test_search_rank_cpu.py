"""The oracle's BeamSearch.search ranks finished hypotheses by a float64 key, also when its costs are float32.

The reference ran under numpy 1.x, where a float32 cost minus ``char_discount * len`` (a Python float) was float64;
lvsr_beam_search_many computes the key in double too.  Under numpy 2 (NEP 50) the same expression is float32, so the
oracle casts the cost to float first.  A replay of the device search keeps its costs in float32, and this pins that
its ranking is still the float64 one."""
from collections import OrderedDict

import numpy as np

from oracle import lvsr_oracle as O

EOL, BIG = 2, 1e4
C_B = np.float32(1000.0)              # finishes at step 0: history [0, C_B], key C_B - 0.2
C_A = np.float32(1000.1)              # finishes at step 1: history [0, 0.5, C_A], key C_A - 0.3


def _computers():
    """Three symbols (eol = 2) whose costs depend only on the last symbol: from the initial symbol, symbol 0 costs
    0.5 and eol C_B; after symbol 0, eol costs C_A - 0.5 (exact in float32, so the history ends at C_A)."""
    def f_logp(att, m, st):
        rows = []
        for y in st["outputs"]:
            rows.append([0.5, BIG, C_B] if y == 3 else [BIG, BIG, np.float32(C_A - np.float32(0.5))])
        return np.asarray(rows, dtype=np.float32)

    def f_next(att, m, st, y):
        return OrderedDict(states=st["states"], outputs=np.asarray(y, dtype=np.int64))

    dummy = np.zeros((1, 1, 1), np.float32)
    return dict(context=lambda x: (dummy, dummy[:, :, 0]),
                initial=lambda att: OrderedDict(states=np.zeros((1, 1), np.float32), outputs=np.array([3])),
                logprobs=f_logp, next=f_next)


def test_ranking_key_is_float64_with_float32_costs():
    # the two keys are equal in float32 arithmetic and 2.4e-5 apart in float64
    assert C_A - 0.3 == C_B - 0.2
    assert float(C_A) - 0.3 < float(C_B) - 0.2
    stats = {}
    done = O.beam_search(None, None, np.zeros((4, 1)), 2, eol_symbol=EOL, max_length=2, char_discount=0.1,
                         computers=_computers(), as_arrays=True, stats=stats)
    assert [list(t) for t, _ in done] == [[3, 0, EOL], [3, EOL]]          # float64: A before B (append order: B, A)
    assert all(c.dtype == np.float32 for _, c in done)
    assert done[0][1][-1] == C_A and done[1][1][-1] == C_B
    assert stats == dict(steps=2, stop=None, finished=2, eol_removed=0, eol_kept_first=0, rejected=0)


def test_counters_of_the_settings():
    """round_to_inf removes the eol hypothesis whose step cost reaches it, ignore_first_eol keeps the step-0 eol in
    the beam, and a validator's rejections are counted."""
    stats = {}
    done = O.beam_search(None, None, np.zeros((4, 1)), 2, eol_symbol=EOL, max_length=2, round_to_inf=999.9,
                         computers=_computers(), as_arrays=True, stats=stats)
    assert [list(t) for t, _ in done] == [[3, 0, EOL]]                # C_B >= 999.9: B is not finished
    assert stats["eol_removed"] == 1 and stats["finished"] == 1
    done = O.beam_search(None, None, np.zeros((4, 1)), 2, eol_symbol=EOL, max_length=2, ignore_first_eol=True,
                         char_discount=0.1, validate_solution_function=lambda rec, seq: len(seq) == 2,
                         computers=_computers(), as_arrays=True, stats=stats)
    assert stats["eol_kept_first"] == 1 and stats["rejected"] >= 1
    assert [list(t) for t, _ in done] == [[3, EOL]]
