"""Float64 oracle of task loss estimation (criterion mse_gain / mse_reward) -- TEST INFRASTRUCTURE ONLY.

With criterion['name'] mse_gain or mse_reward the reference's emitter is RewardRegressionEmitter
(lvsr/bricks/__init__.py:119-202, lvsr/bricks/recognizer.py:285-297).  Everything else is oracle/lvsr_oracle.py's;
only what the emitter changes is restated here:

  * RewardOp(groundtruth, prediction) (lvsr/ops.py:236-294 over lvsr/error_rate.py:11-112): per utterance, the
    groundtruth is cut after its first eos (it must then end in eos), the prediction likewise; D = the edit distance
    matrix, R[j, c] = -min(min_i D[i, j] + 1, min over i < len(g), g[i] = c of D[i, j]), R[j, eos] = -D[len(g)-1, j];
    G[0] = R[0], G[j] = R[j] - R[j-1, y[j-1]].  Rows past the cut prediction hold reward -1, gain -1000;
  * the cost (the labels being their own groundtruth unless analyze substitutes it): mse_gain
    sum_v (r - max(G, min_reward))^2, mse_reward sum_v (r + cumsum([0, r[1:, y_1:]]) - R)^2, times the label mask;
  * the emitter: costs -readouts (no log-softmax), emit = arg-max of the readouts, initial output 0.
"""
from collections import OrderedDict

import numpy as np

from oracle import lvsr_oracle as O


def edit_distance_matrix(g, y):
    """_edit_distance_matrix's dist (lvsr/error_rate.py:11-55): D[i, j] between g[:i] and y[:j]."""
    D = np.zeros((len(g) + 1, len(y) + 1), dtype=np.int64)
    D[:, 0] = np.arange(len(g) + 1)
    D[0, :] = np.arange(len(y) + 1)
    for i in range(1, len(g) + 1):
        for j in range(1, len(y) + 1):
            D[i, j] = min(D[i - 1, j] + 1, D[i, j - 1] + 1, D[i - 1, j - 1] + (g[i - 1] != y[j - 1]))
    return D


def reward_matrix(g, y, V, eos):
    """reward_matrix (lvsr/error_rate.py:79-103): [len(y) + 1, V]."""
    g, y = list(g), list(y)
    if not g or g[-1] != eos:
        raise ValueError("Last character of the groundtruth must be EOS")
    D = edit_distance_matrix(g, y)
    opt = D.min(axis=0)
    best = np.repeat(opt[:, None] + 1, V, axis=1)
    for i in range(len(g)):
        best[:, g[i]] = np.minimum(best[:, g[i]], D[i, :])
    best[:, eos] = D[len(g) - 1, :]
    return -best


def gain_matrix(g, y, V, eos, rewards=None):
    """gain_matrix (lvsr/error_rate.py:105-112): [len(y) + 1, V]."""
    R = reward_matrix(g, y, V, eos) if rewards is None else rewards
    G = R.copy()
    G[1:] -= R[:-1][np.arange(len(y)), list(y)][:, None]
    return G


def _cut(seq, eos):
    seq = list(seq)
    return seq[:seq.index(eos) + 1] if eos in seq else seq


def reward_op(groundtruth, prediction, V, eos):
    """RewardOp.perform (lvsr/ops.py:244-285): groundtruth [Lg, B], prediction [L, B] -> rewards, gains [L, B, V]."""
    groundtruth, prediction = np.asarray(groundtruth), np.asarray(prediction)
    L, B = prediction.shape
    rewards = np.empty((L, B, V))
    gains = np.empty((L, B, V))
    for b in range(B):
        g = _cut(groundtruth[:, b], eos)
        y = _cut(prediction[:, b], eos)
        R = reward_matrix(g, y, V, eos)
        G = gain_matrix(g, y, V, eos, R)
        rewards[:, b] = -1
        gains[:, b] = -1000
        rewards[:len(y), b] = R[:-1]
        gains[:len(y), b] = G[:-1]
    return rewards, gains


def tle_cost(name, readouts, outputs, rewards, gains, min_reward, mask=None):
    """RewardRegressionEmitter.cost for readouts [L, B, V] (lvsr/bricks/__init__.py:135-184) times the mask."""
    readouts = np.asarray(readouts, dtype=np.float64)
    if name == "mse_gain":
        cost = ((readouts - np.maximum(gains, min_reward)) ** 2).sum(axis=-1)
    elif name == "mse_reward":
        picked = np.take_along_axis(readouts, np.asarray(outputs)[..., None], axis=-1)[..., 0]
        picked[0] = 0
        predicted = readouts + picked.cumsum(axis=0)[:, :, None]
        cost = ((predicted - rewards) ** 2).sum(axis=-1)
    else:
        raise ValueError(name)
    return cost if mask is None else cost * mask


def readouts(cfg, params, attended, attended_mask, labels, labels_mask=None):
    """The teacher-forced readouts [L, B, V] (O.cost_matrix's, before the emitter)."""
    r = O.cost_matrix(cfg, params, attended, attended_mask, labels, labels_mask, return_all=True)
    return O.readout(cfg, params, r["states"], r["weighted_averages"]), r


def cost_matrix(cfg, params, attended, attended_mask, labels, labels_mask, criterion, groundtruth=None,
                return_all=False):
    """generator.cost_matrix under RewardRegressionEmitter; criterion = dict(name, min_reward=-1.0)."""
    ro, r = readouts(cfg, params, attended, attended_mask, labels, labels_mask)
    g = labels if groundtruth is None else groundtruth
    rewards, gains = reward_op(g, labels, cfg["num_phonemes"], cfg["eos_label"])
    costs = tle_cost(criterion["name"], ro, labels, rewards, gains, criterion.get("min_reward", -1.0), labels_mask)
    if return_all:
        return dict(r, costs=costs, readouts=ro)
    return costs


def initial_states(cfg, params, batch_size, attended):
    """O.initial_states with RewardRegressionEmitter.initial_outputs = 0."""
    st = O.initial_states(cfg, params, batch_size, attended)
    st["outputs"] = np.zeros((batch_size,), dtype=np.int64)
    return st


def emitter_costs(cfg, params, attended, attended_mask, st):
    """RewardRegressionEmitter.costs (lvsr/bricks/__init__.py:194-196): -readouts."""
    wa, _, _, _ = O.take_glimpses(cfg, params, attended, None, attended_mask, st["weights"], st["step"], st["states"])
    return -O.readout(cfg, params, st["states"], wa)


def generate_greedy(cfg, params, attended, attended_mask, n_steps):
    """generate() with RewardRegressionEmitter: emit = arg-max of the readouts, cost = the emitted readout."""
    B = attended.shape[1]
    st = initial_states(cfg, params, B, attended)
    outs, costs = [], []
    for _ in range(n_steps):
        c = emitter_costs(cfg, params, attended, attended_mask, st)
        y = c.argmin(axis=1)
        costs.append(-c[np.arange(B), y])
        st = O.next_state_computer(cfg, params, attended, attended_mask, st, y)
        outs.append(y)
    return np.stack(outs), np.stack(costs), st


def beam_search(cfg, params, recordings, beam_size, **kw):
    """O.beam_search on the TLE emitter's costs and initial output."""
    computers = OrderedDict(initial=lambda att: initial_states(cfg, params, 1, att),
                            logprobs=lambda att, m, st: emitter_costs(cfg, params, att, m, st))
    return O.beam_search(cfg, params, recordings, beam_size, computers=computers, **kw)
