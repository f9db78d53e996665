"""Float64 gradient oracle of task-loss-estimation training (criterion mse_gain / mse_reward) -- TEST INFRASTRUCTURE
ONLY.

The training cost of the reference under RewardRegressionEmitter is sum(cost_matrix) / B (lvsr/main.py:340-345) with
cost_matrix = tests/tle_oracle.py's: the teacher-forced readouts of the prediction, no log-softmax, and the mse_gain /
mse_reward loss against RewardOp's matrices, which hold no parameter.  The prediction is (lvsr/main.py:245-283):

  * imitative exploration: the labels, with their mask, as their own groundtruth;
  * greedy exploration: L + 10 steps of generate() (the arg-max of the readouts, fed back), masked by
    prediction_mask below, scored against the labels as groundtruth.  No gradient flows through the generation.

The torch float64 mirror restates the teacher-forced readouts with G's glimpses and GRU step (content attention:
content_oracle's loop) and readout_oracle's readout, which takes any post-merge depth, then tle_oracle's loss.  The
encoder is G's, or unidirectional_oracle's for a forward-only one (bidir False), behind bottom_oracle's MLP when the
config has one.  tests/test_tle_train_cpu.py pins it against tle_oracle.cost_matrix and central differences of the
numpy oracle.
"""
from collections import OrderedDict

import numpy as np

import readout_oracle as RO
import tle_oracle as TO
from oracle import lvsr_oracle_grad as G

EXTRA_STEPS = 10            # lvsr/main.py:251: length_expand


def prediction_mask(prediction, eos):
    """add_exploration's mask (lvsr/main.py:252-258): lt(cumsum(eq(prediction, eos)), 1), rolled by one step along
    time, with row 0 set to ones."""
    m = (np.cumsum(np.asarray(prediction) == eos, axis=0) < 1).astype(np.float64)
    m = np.roll(m, 1, axis=0)
    m[0] = 1
    return m


def _encode_torch(cfg, p, x, mask):
    """(attended, attended_mask, the config the decoder functions read) of recordings x [T, B, F]."""
    import bottom_oracle as BO
    import unidirectional_oracle as U
    if cfg.get("bottom") and cfg["bottom"]["dims"]:
        x = BO._bottom_torch(cfg, p, x)
        cfg = BO.inner(cfg)
    if cfg.get("bidir", True) is False:
        attended, amask = U._encoder_torch(cfg, p, x, mask)
        return attended, amask, U.decoder_config(cfg)
    attended, amask = G._encoder(cfg, p, x, mask)
    return attended, amask, cfg


def _readouts_torch(cfg, p, attended, attended_mask, labels, labels_mask):
    """The teacher-forced readouts [L, B, V] of `labels` (G._cost_matrix's loop before its log-softmax)."""
    import torch
    if cfg.get("attention_type") == "content":
        import content_oracle as CO
        kept = []

        def readout(cfg_, p_, states, wavg):
            kept.append(RO.readout_torch(cfg_, p_, states, wavg))
            return kept[-1]
        CO._cost_matrix_torch(cfg, p, attended, attended_mask, labels, labels_mask, readout=readout)
        return kept[0]
    L, B = labels.shape
    P = attended @ p[G._ATT + "/preprocess.W"] + p[G._ATT + "/preprocess.b"]
    if cfg.get("embed_outputs", True):
        fb = p[G._GEN + "/readout/lookupfeedback/lookuptable.W"][torch.as_tensor(labels)]
    else:
        fb = torch.eye(cfg["num_phonemes"] + 1, dtype=attended.dtype)[torch.as_tensor(labels)]
    inputs = fb @ p[G._GEN + "/fork/fork_inputs.W"] + p[G._GEN + "/fork/fork_inputs.b"]
    gate_inputs = fb @ p[G._GEN + "/fork/fork_gate_inputs.W"] + p[G._GEN + "/fork/fork_gate_inputs.b"]
    s = p[G._TR + "/transition.initial_state"][None, :].expand(B, -1)
    w = torch.zeros((B, attended.shape[0]), dtype=attended.dtype)
    w[:, 0] = 1
    step = np.zeros((B,), dtype=np.int64)
    prev, ctxs = [], []
    for i in range(L):
        prev.append(s)
        wavg, w, step = G._take_glimpses(cfg, p, attended, P, attended_mask, w, step, s)
        a = wavg @ p[G._TR + "/distribute/fork_inputs.W"] + inputs[i]
        g = wavg @ p[G._TR + "/distribute/fork_gate_inputs.W"] + gate_inputs[i]
        s = G._gru_step(s, a, g, p[G._TR + "/transition.state_to_state"], p[G._TR + "/transition.state_to_gates"],
                        None if labels_mask is None else labels_mask[i])
        ctxs.append(wavg)
    return RO.readout_torch(cfg, p, torch.stack(prev), torch.stack(ctxs))


def tle_cost_torch(name, readouts, outputs, rewards, gains, min_reward, mask=None):
    """mirror of TO.tle_cost."""
    import torch
    rewards = torch.as_tensor(rewards, dtype=torch.float64)
    gains = torch.as_tensor(gains, dtype=torch.float64)
    if name == "mse_gain":
        cost = ((readouts - torch.clamp(gains, min=min_reward)) ** 2).sum(dim=-1)
    elif name == "mse_reward":
        picked = torch.gather(readouts, 2, torch.as_tensor(np.asarray(outputs))[..., None])[..., 0]
        picked = torch.cat([torch.zeros_like(picked[:1]), picked[1:]])
        cost = ((readouts + picked.cumsum(dim=0)[:, :, None] - rewards) ** 2).sum(dim=-1)
    else:
        raise ValueError(name)
    return cost if mask is None else cost * mask


def cost_matrix_torch(cfg, p, attended, attended_mask, labels, labels_mask, criterion, groundtruth=None):
    """mirror of TO.cost_matrix: the loss rows [L, B] of the prediction `labels` against `groundtruth` (None: the
    labels)."""
    ro = _readouts_torch(cfg, p, attended, attended_mask, labels, labels_mask)
    g = labels if groundtruth is None else groundtruth
    rewards, gains = TO.reward_op(g, labels, cfg["num_phonemes"], cfg["eos_label"])
    return tle_cost_torch(criterion["name"], ro, labels, rewards, gains, criterion.get("min_reward", -1.0), labels_mask)


def cost_and_grads(cfg, params, recordings, recordings_mask, labels, labels_mask, criterion, groundtruth=None):
    """sum(cost_matrix) / B of the prediction `labels` (mask `labels_mask`) against `groundtruth` and its float64
    gradient: (cost, OrderedDict name -> ndarray)."""
    import torch
    p = OrderedDict((k, torch.tensor(np.asarray(v, dtype=np.float64), requires_grad=True)) for k, v in params.items())
    x = torch.as_tensor(np.asarray(recordings, dtype=np.float64))
    m = None if recordings_mask is None else torch.as_tensor(np.asarray(recordings_mask, dtype=np.float64))
    lm = None if labels_mask is None else torch.as_tensor(np.asarray(labels_mask, dtype=np.float64))
    labels = np.asarray(labels, dtype=np.int64)
    attended, amask, dcfg = _encode_torch(cfg, p, x, m)
    costs = cost_matrix_torch(dcfg, p, attended, amask, labels, lm, criterion, groundtruth)
    cost = costs.sum() / labels.shape[1]
    grads = torch.autograd.grad(cost, list(p.values()), allow_unused=True)
    return float(cost.detach()), OrderedDict((k, np.zeros(v.shape) if g is None else g.numpy().copy())
                                             for (k, v), g in zip(p.items(), grads))


def train_step(cfg, params, state, batch, tc, criterion):
    """One imitative update: the gradient above, then G's step rules."""
    cost, grads = cost_and_grads(cfg, params, *batch, criterion=criterion)
    p64 = OrderedDict((k, np.asarray(v, dtype=np.float64)) for k, v in params.items())
    steps = G.apply_step_rules(p64, grads, state, tc)
    return OrderedDict((k, p64[k] - steps[k]) for k in p64), cost, grads


def greedy_readouts(cfg, params, recordings, recordings_mask, prediction):
    """The readouts [n, B, V] generate() sees along `prediction`: its state is fed the previous picks without a mask,
    so they are the teacher-forced readouts of the prediction, unmasked."""
    import torch
    p = OrderedDict((k, torch.as_tensor(np.asarray(v, dtype=np.float64))) for k, v in params.items())
    x = torch.as_tensor(np.asarray(recordings, dtype=np.float64))
    m = None if recordings_mask is None else torch.as_tensor(np.asarray(recordings_mask, dtype=np.float64))
    with torch.no_grad():
        attended, amask, dcfg = _encode_torch(cfg, p, x, m)
        return _readouts_torch(dcfg, p, attended, amask, np.asarray(prediction, dtype=np.int64), None).numpy()


def check_greedy(readouts, prediction, noise):
    """Every pick of `prediction` [n, B] is the arg-max of the oracle's readouts on its own prefix, unless the best
    readout leads the pick's by less than `noise` (float32 can order them either way).  Returns the number of such
    near ties."""
    n, B = prediction.shape
    ties = 0
    for t in range(n):
        for b in range(B):
            r = readouts[t, b]
            y = int(prediction[t, b])
            best = int(np.argmax(r))
            if y != best:
                assert r[best] - r[y] <= noise, (t, b, y, best, r[best] - r[y])
                ties += 1
    return ties
