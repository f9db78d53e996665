"""Float64 oracle of task loss estimation with an FST language model (criterion mse_gain / mse_reward with net.lm)
-- TEST INFRASTRUCTURE ONLY.  It composes tests/tle_oracle.py and tests/lm_oracle.py the way the reference composes
their bricks (lvsr/bricks/recognizer.py:285-338):

  * the emitter stays RewardRegressionEmitter; only SoftmaxEmitter would have become LMEmitter.  The readout becomes
    ShallowFusionReadout over the TLE readouts r (the logits, no softmax):
      x = [tot] ( [am] log_softmax(am_beta r) + weight [lm] log_softmax(-lm_add) )   (language_models.py:74-104);
  * the emitter costs (logprobs, beam search) are -x, the row the log-likelihood emitter writes under fusion; the
    initial output stays 0;
  * cost / analyze apply RewardRegressionEmitter.cost to x: mse_gain sum_v (x - max(G, min_reward))^2, mse_reward
    with its cumulative sum over the picked x.  R and G are RewardOp's of the groundtruth against the prediction, while
    the LM rows follow the labels fed in (the prediction): the quirk this oracle keeps;
  * greedy generation emits the arg-max of x with cost x[picked], and each row's LM state advances by its symbol.
"""
from collections import OrderedDict

import numpy as np

import lm_oracle as LO
import tle_oracle as TO
from oracle import lvsr_oracle as O


def fused_readouts(logits, add, o):
    """ShallowFusionReadout.readout of the TLE readouts: x [.., V] (o: the lm options, as lm_oracle takes them)."""
    return -LO.fused_costs(logits, add, o)


def loss(criterion, x, labels, groundtruth, V, eos, mask=None):
    """RewardRegressionEmitter.cost of the fused readouts x [L, B, V] for the prediction `labels` [L, B] scored against
    `groundtruth` [Lg, B] (None: the labels), times the mask; criterion = dict(name, min_reward=-1.0)."""
    g = labels if groundtruth is None else groundtruth
    rewards, gains = TO.reward_op(g, labels, V, eos)
    return TO.tle_cost(criterion["name"], x, labels, rewards, gains, criterion.get("min_reward", -1.0), mask)


def cost_of_logits(cfg, fst, o, criterion, logits, labels, labels_mask=None, groundtruth=None):
    """The TLE + LM cost matrix [L, B] from teacher-forced logits [L, B, V]: the LM rows along the labels, then loss."""
    V = cfg["num_phonemes"]
    add = LO.lm_path(fst, labels, labels_mask, V, o["no_transition_cost"])
    return loss(criterion, fused_readouts(logits, add, o), labels, groundtruth, V, cfg["eos_label"], labels_mask)


def cost_matrix(cfg, params, fst, o, attended, attended_mask, labels, labels_mask, criterion, groundtruth=None,
                oracle=O, return_all=False):
    """generator.cost_matrix under RewardRegressionEmitter with shallow fusion (`oracle`: the attention's oracle)."""
    r = oracle.cost_matrix(cfg, params, attended, attended_mask, labels, labels_mask, return_all=True)
    logits = O.readout(cfg, params, r["states"], r["weighted_averages"])
    V = cfg["num_phonemes"]
    add = LO.lm_path(fst, labels, labels_mask, V, o["no_transition_cost"])
    x = fused_readouts(logits, add, o)
    costs = loss(criterion, x, labels, groundtruth, V, cfg["eos_label"], labels_mask)
    if return_all:
        return dict(r, costs=costs, logits=logits, add=add, readouts=x)
    return costs


def emitter_costs(cfg, params, o, attended, attended_mask, st, oracle=O):
    """RewardRegressionEmitter.costs of the fused readouts: -x for the rows of st (whose lm_add is their LM row)."""
    wa, _, _, _ = oracle.take_glimpses(cfg, params, attended, None, attended_mask, st["weights"], st["step"],
                                       st["states"])
    return LO.fused_costs(O.readout(cfg, params, st["states"], wa), st["lm_add"], o)


def _lm_rows(fst, sets, ys, V, ntc):
    out_sets, rows = [], []
    for s, y in zip(sets, ys):
        s2, row = LO.next_state(fst, s, y, V, ntc)
        out_sets.append(s2)
        rows.append(row)
    arr = np.empty(len(out_sets), dtype=object)
    arr[:] = out_sets
    return arr, (np.stack(rows) if rows else np.zeros((0, V), np.float32))


def initial_states(cfg, params, fst, o, batch_size, attended, oracle=O):
    """The TLE initial states (output 0) with every row's LM set and cost row."""
    st = oracle.initial_states(cfg, params, batch_size, attended)
    st["outputs"] = np.zeros((batch_size,), dtype=np.int64)
    s, row = LO.initial(fst, cfg["num_phonemes"], o["no_transition_cost"])
    sets = np.empty(batch_size, dtype=object)
    sets[:] = [dict(s) for _ in range(batch_size)]
    st["lm_sets"] = sets
    st["lm_add"] = np.repeat(row[None, :], batch_size, axis=0)
    return st


def next_states(cfg, params, fst, o, attended, attended_mask, st, y, oracle=O):
    nxt = oracle.next_state_computer(cfg, params, attended, attended_mask,
                                     OrderedDict((k, v) for k, v in st.items() if not k.startswith("lm_")), y)
    nxt["lm_sets"], nxt["lm_add"] = _lm_rows(fst, st["lm_sets"], y, cfg["num_phonemes"], o["no_transition_cost"])
    return nxt


def generate_greedy(cfg, params, fst, o, attended, attended_mask, n_steps, oracle=O):
    """generate() with RewardRegressionEmitter over fused readouts: outputs [n, B], costs [n, B] = the emitted x."""
    B = attended.shape[1]
    st = initial_states(cfg, params, fst, o, B, attended, oracle)
    outs, costs = [], []
    for _ in range(n_steps):
        c = emitter_costs(cfg, params, o, attended, attended_mask, st, oracle)
        y = c.argmin(axis=1)
        costs.append(-c[np.arange(B), y])
        st = next_states(cfg, params, fst, o, attended, attended_mask, st, y, oracle)
        outs.append(y)
    return np.stack(outs), np.stack(costs), st


def computers(cfg, params, fst, o):
    """initial / logprobs / next for O.beam_search: the TLE emitter over fused readouts, the LM state in the dict."""
    return dict(initial=lambda att: initial_states(cfg, params, fst, o, 1, att),
                logprobs=lambda att, m, st: emitter_costs(cfg, params, o, att, m, st),
                next=lambda att, m, st, y: next_states(cfg, params, fst, o, att, m, st, y))


def beam_search(cfg, params, fst, o, recordings, beam_size, **kw):
    """O.beam_search on the fused TLE emitter costs."""
    return O.beam_search(cfg, params, recordings, beam_size, computers=computers(cfg, params, fst, o), **kw)
