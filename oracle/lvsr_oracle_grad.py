"""Gradient + optimizer oracle for the training step (SURVEY.md 8 row a21 / f1) -- TEST INFRASTRUCTURE ONLY.

What the reference does for one training step (lvsr/main.py:340-345,480-519;
libs/blocks/blocks/algorithms/__init__.py:244-256,284-287):

    cost      = sum(cost_matrix) / batch_size                       lvsr/main.py:340-345
    gradients = theano.tensor.grad(cost, parameters)                B/algorithms/__init__.py:218-225
    steps     = CompositeRule([StepClipping, Momentum?, AdaDelta?, Restrict(VariableClipping(axis=0), WEIGHT)?,
                               RemoveNotFinite(0.0), BurnIn?])      lvsr/main.py:480-519
    parameter <- parameter - step                                   B/algorithms/__init__.py:249-251

Theano's symbolic differentiation is restated here with torch.float64 autograd on the CPU over a
torch re-statement of the forward pass that mirrors oracle/lvsr_oracle.py line by line (each function
names the numpy function it mirrors; tests/test_oracle_grad.py pins the mirror: forward equality to
1e-12 against the numpy oracle for every prior / normaliser, and central finite differences of the
numpy oracle's cost against the autograd gradient).  The step rules are plain numpy and are pinned by
the reference's own literals (libs/blocks/tests/algorithms/test_algorithms.py:80-119,182-249,312-349).

Nothing under attention-lvcsr_b200/ imports this file.
"""
from __future__ import annotations

from collections import OrderedDict

import numpy as np

from . import lvsr_oracle as O

_ATT = O._ATT
_GEN = O._GEN
_TR = O._TR


def _torch():
    import torch
    return torch


# --------------------------------------------------------------------------
# forward pass in torch.float64 (mirror of oracle/lvsr_oracle.py)
# --------------------------------------------------------------------------


def _gru_step(h, inputs, gate_inputs, Ws, Wg, mask):
    """mirror of O.gru_step (B/bricks/recurrent.py:608-620)."""
    torch = _torch()
    D = h.shape[-1]
    g = torch.sigmoid(h @ Wg + gate_inputs)
    z, r = g[:, :D], g[:, D:]
    c = torch.tanh((h * r) @ Ws + inputs)
    nxt = c * z + h * (1 - z)
    if mask is not None:
        nxt = mask[:, None] * nxt + (1 - mask[:, None]) * h
    return nxt


def _encoder(cfg, p, x, mask):
    """mirror of O.encoder / O.bidirectional / O.recurrent_with_fork (lvsr/bricks/__init__.py:28-43,71-78)."""
    torch = _torch()
    for l, k in enumerate(cfg["subsample"]):
        outs = []
        for d, reverse in (("forward", False), ("backward", True)):
            base = "/recognizer/encoder/bidir%d/%s" % (l, d)
            a = x @ p[base + "/fork/fork_inputs.W"] + p[base + "/fork/fork_inputs.b"]
            g = x @ p[base + "/fork/fork_gate_inputs.W"] + p[base + "/fork/fork_gate_inputs.b"]
            T, B = x.shape[0], x.shape[1]
            h = p[base + "/gatedrecurrent.initial_state"][None, :].expand(B, -1)
            seq = [None] * T
            order = range(T - 1, -1, -1) if reverse else range(T)
            for t in order:
                h = _gru_step(h, a[t], g[t], p[base + "/gatedrecurrent.state_to_state"],
                              p[base + "/gatedrecurrent.state_to_gates"], None if mask is None else mask[t])
                seq[t] = h            # Bidirectional re-reverses the backward scan (recurrent.py:655-663)
            outs.append(torch.stack(seq))
        x = torch.cat(outs, dim=2)[::k]
        if mask is not None:
            mask = mask[::k]
    enc_mask = mask if mask is not None else torch.ones_like(x[:, :, 0])
    return x, enc_mask


def _compute_weights(e, mask, normalizer):
    """mirror of O.compute_weights (lvsr/bricks/attention.py:191-213)."""
    torch = _torch()
    if normalizer == "softmax":
        e = e - e.max(dim=0).values
        un = torch.exp(e)
    elif normalizer == "logistic":
        un = torch.sigmoid(e)
    elif normalizer == "relu":
        un = torch.clamp(e / 1000.0, min=0.0)
    else:
        raise ValueError(normalizer)
    un = un * mask
    norm = un.sum(dim=0) + (mask.sum(dim=0) == 0).to(e.dtype)
    return un / norm


def _take_glimpses(cfg, p, attended, P, attended_mask, weights, step, states):
    """mirror of O.take_glimpses / O.compute_energies (lvsr/bricks/attention.py:98-183).  The window
    comes from the numpy oracle on detached values: floor / argmax / comparisons carry no gradient in
    Theano either (and the median position is an explicit disconnected_grad, attention.py:143-144)."""
    torch = _torch()
    length = attended.shape[0]
    begin, end, add_mask = O.attention_window(cfg, length, weights.detach().numpy(), step)
    n = cfg["conv_n"]
    att_cut, P_cut = attended[begin:end], P[begin:end]
    mask_cut = attended_mask[begin:end]
    if add_mask is not None:
        mask_cut = mask_cut * torch.as_tensor(add_mask.T)
    w_cut = weights[:, begin:end]
    match = P_cut + (states @ p[_ATT + "/state_trans/transform_states.W"])[None]
    filt = p[_ATT + "/conv1d.filters"]                                        # [K, 2n+1]
    # true convolution, full mode, centre crop [n:-n]  ==  cross-correlation with the flipped filter, padding n
    conv = torch.nn.functional.conv1d(w_cut[:, None, :], torch.flip(filt, dims=[1])[:, None, :], padding=n)   # [B,K,Tw]
    match = match + (conv.permute(0, 2, 1) @ p[_ATT + "/handler.W"]).permute(1, 0, 2)
    e = (torch.tanh(match) @ p[_ATT + "/energy_comp/linear.W"])[..., 0]
    if cfg["energy_normalizer"] != "softmax":
        e = e + p[_ATT + "/energy_comp/linear.b"][0]
    w = _compute_weights(e, mask_cut, cfg["energy_normalizer"])
    wavg = (w[:, :, None] * att_cut).sum(dim=0)
    new_w = torch.zeros_like(weights.T)
    new_w = torch.cat([new_w[:begin], w, new_w[end:]], dim=0)
    return wavg, new_w.T, step + 1


def _cost_matrix(cfg, p, attended, attended_mask, labels, labels_mask):
    """mirror of O.cost_matrix (B/bricks/sequence_generators.py:254-326)."""
    torch = _torch()
    L, B = labels.shape
    P = attended @ p[_ATT + "/preprocess.W"] + p[_ATT + "/preprocess.b"]
    if cfg.get("embed_outputs", True):
        fb = p[_GEN + "/readout/lookupfeedback/lookuptable.W"][torch.as_tensor(labels)]
    else:
        fb = torch.eye(cfg["num_phonemes"] + 1, dtype=attended.dtype)[torch.as_tensor(labels)]
    inputs = fb @ p[_GEN + "/fork/fork_inputs.W"] + p[_GEN + "/fork/fork_inputs.b"]
    gate_inputs = fb @ p[_GEN + "/fork/fork_gate_inputs.W"] + p[_GEN + "/fork/fork_gate_inputs.b"]
    s = p[_TR + "/transition.initial_state"][None, :].expand(B, -1)
    w = torch.zeros((B, attended.shape[0]), dtype=attended.dtype)
    w[:, 0] = 1
    step = np.zeros((B,), dtype=np.int64)
    prev, ctxs = [], []
    for i in range(L):
        prev.append(s)
        wavg, w, step = _take_glimpses(cfg, p, attended, P, attended_mask, w, step, s)
        a = wavg @ p[_TR + "/distribute/fork_inputs.W"] + inputs[i]
        g = wavg @ p[_TR + "/distribute/fork_gate_inputs.W"] + gate_inputs[i]
        s = _gru_step(s, a, g, p[_TR + "/transition.state_to_state"], p[_TR + "/transition.state_to_gates"],
                      None if labels_mask is None else labels_mask[i])
        ctxs.append(wavg)
    prev, ctx = torch.stack(prev), torch.stack(ctxs)
    r = ctx @ p[_GEN + "/readout/merge/transform_weighted_averages.W"]
    if cfg["use_states_for_readout"]:
        r = r + prev @ p[_GEN + "/readout/merge/transform_states.W"]
    r = r + p[_GEN + "/readout/post_merge/bias.b"]
    act = cfg["post_merge_activation"]
    if act == "maxout":
        pieces = cfg["maxout_pieces"]
        r = r.reshape(r.shape[:-1] + (r.shape[-1] // pieces, pieces)).max(dim=-1).values
    elif act == "relu":
        r = torch.clamp(r, min=0)
    elif act == "tanh":
        r = torch.tanh(r)
    r = r @ p[_GEN + "/readout/post_merge/mlp/linear_0.W"] + p[_GEN + "/readout/post_merge/mlp/linear_0.b"]
    logp = torch.log_softmax(r, dim=-1)
    costs = -torch.gather(logp, 2, torch.as_tensor(labels)[..., None])[..., 0]
    if labels_mask is not None:
        costs = costs * labels_mask
    return costs


WEIGHT_LEAVES = ("W", "state_to_state", "state_to_gates")


def is_weight(name):
    """Parameters carrying the WEIGHT role, the ones VariableFilter(roles=[WEIGHT]) selects for the decay term and
    the max-norm subjects (lvsr/main.py:418-420,493): every Linear / LookupTable W (B/bricks/simple.py:49,
    B/bricks/lookup.py:42) and the recurrent matrices (B/bricks/recurrent.py:556,560).  Not biases, not initial
    states, and not the conv filters: Conv1D._allocate (lvsr/bricks/attention.py:31-33) adds no role, so they carry
    only the PARAMETER role every brick parameter gets (B/bricks/base.py:36-44)."""
    return name.rsplit(".", 1)[1] in WEIGHT_LEAVES


def cost_and_grads(cfg, params, recordings, recordings_mask, labels, labels_mask, decay=0.0, return_costs=False):
    """train_cost = sum(costs) / B (+ decay * ||WEIGHT parameters||^2, lvsr/main.py:419-421) and its gradient
    with respect to every parameter, float64.  -> (cost, OrderedDict name -> ndarray)."""
    torch = _torch()
    p = OrderedDict((k, torch.tensor(np.asarray(v, dtype=np.float64), requires_grad=True)) for k, v in params.items())
    x = torch.as_tensor(np.asarray(recordings, dtype=np.float64))
    m = None if recordings_mask is None else torch.as_tensor(np.asarray(recordings_mask, dtype=np.float64))
    lm = None if labels_mask is None else torch.as_tensor(np.asarray(labels_mask, dtype=np.float64))
    labels = np.asarray(labels, dtype=np.int64)
    attended, amask = _encoder(cfg, p, x, m)
    costs = _cost_matrix(cfg, p, attended, amask, labels, lm)
    cost = costs.sum() / labels.shape[1]
    if decay > 0:
        cost = cost + decay * sum((v ** 2).sum() for k, v in p.items() if is_weight(k))
    grads = torch.autograd.grad(cost, list(p.values()), allow_unused=True)
    out = OrderedDict()
    for (k, v), g in zip(p.items(), grads):
        out[k] = np.zeros(v.shape) if g is None else g.numpy().copy()
    if return_costs:
        return float(cost.detach()), out, costs.detach().numpy()
    return float(cost.detach()), out


# --------------------------------------------------------------------------
# step rules (B/algorithms/__init__.py), plain numpy
# --------------------------------------------------------------------------


def l2_norm(arrays):
    """B/theano_expressions.py l2_norm: sqrt of the sum of squares over all tensors."""
    return float(np.sqrt(sum(float((np.asarray(a, dtype=np.float64) ** 2).sum()) for a in arrays)))


def step_clipping(steps, threshold):
    """StepClipping.compute_steps, B/algorithms/__init__.py:634-643: multiplier = 1 if norm < threshold
    else threshold / norm (one norm over ALL steps)."""
    if not threshold:
        return steps
    norm = l2_norm(steps.values())
    mult = 1.0 if norm < threshold else threshold / norm
    return OrderedDict((k, v * mult) for k, v in steps.items())


def momentum(steps, state, learning_rate, mom):
    """Momentum = CompositeRule([Scale(lr), BasicMomentum(m)]), :400,423-428,431-461:
    step = m * velocity + lr * previous_step; velocity <- step."""
    out = OrderedDict()
    for k, v in steps.items():
        vel = state.setdefault("velocity", {}).get(k, np.zeros_like(v))
        s = mom * vel + learning_rate * v
        state["velocity"][k] = s
        out[k] = s
    return out


def adadelta(steps, state, decay_rate, epsilon):
    """AdaDelta.compute_step, :490-516."""
    out = OrderedDict()
    for k, g in steps.items():
        ms_step = state.setdefault("mean_square_step", {}).get(k, np.zeros_like(g))
        ms_dx = state.setdefault("mean_square_delta_x", {}).get(k, np.zeros_like(g))
        ms_step_t = decay_rate * ms_step + (1 - decay_rate) * g ** 2
        dx = np.sqrt(ms_dx + epsilon) / np.sqrt(ms_step_t + epsilon) * g
        state["mean_square_step"][k] = ms_step_t
        state["mean_square_delta_x"][k] = decay_rate * ms_dx + (1 - decay_rate) * dx ** 2
        out[k] = dx
    return out


def variable_clipping(parameter, step, threshold, axis=None):
    """VariableClipping.compute_step, :701-720: clip the norm of (parameter - step) along `axis`
    (None: the whole tensor) and return the equivalent step."""
    new = parameter - step
    if axis is None:
        norms = np.sqrt((new ** 2).sum())
    else:
        axes = tuple(sorted(set((axis,) if np.isscalar(axis) else tuple(axis))))
        if any(a >= new.ndim for a in axes):
            raise ValueError("Invalid axis %s for ndim=%d" % (axes, new.ndim))
        norms = np.sqrt((new ** 2).sum(axis=axes, keepdims=True))
    with np.errstate(divide="ignore", invalid="ignore"):
        shrinking = parameter - (threshold / norms) * new
    return np.where(norms > threshold, shrinking, step)


def remove_not_finite(parameter, step, scaler=1.0):
    """RemoveNotFinite.compute_step, :855-861.  NOTE lvsr passes scaler=0.0 (lvsr/main.py:516): a step with
    a non-finite SUM becomes the parameter itself, i.e. the parameter is ZEROED (the comment in main.py
    says "not changed at all"; the code does this)."""
    s = np.sum(step)
    if np.isnan(s) or np.isinf(s):
        return (1 - scaler) * parameter
    return step


def make_train_config(gradient_threshold=10.0, rules=("momentum", "adadelta"), scale=1.0, momentum=0.0,
                      decay_rate=0.95, epsilon=1e-8, max_norm=1.0, burn_in_steps=0, decay=0.0):
    """config['training'] / config['regularization'] keys read by lvsr/main.py:480-519 (defaults: wsj_jan_new.yaml:75-85)."""
    return dict(gradient_threshold=gradient_threshold, rules=tuple(rules), scale=scale, momentum=momentum,
                decay_rate=decay_rate, epsilon=epsilon, max_norm=max_norm, burn_in_steps=burn_in_steps, decay=decay)


def apply_step_rules(params, grads, state, tc):
    """The CompositeRule of lvsr/main.py:509-516 applied to `grads`; returns the steps and updates `state`
    (velocities, AdaDelta accumulators, remaining burn-in steps) in place."""
    steps = OrderedDict((k, np.asarray(g, dtype=np.float64)) for k, g in grads.items())
    steps = step_clipping(steps, tc["gradient_threshold"])
    if "momentum" in tc["rules"]:
        steps = momentum(steps, state, tc["scale"], tc["momentum"])
    if "adadelta" in tc["rules"]:
        steps = adadelta(steps, state, tc["decay_rate"], tc["epsilon"])
    if tc.get("max_norm", 0) and tc["max_norm"] > 0:
        steps = OrderedDict((k, variable_clipping(params[k], s, tc["max_norm"], axis=0) if (is_weight(k) and s.ndim >= 1) else s)
                            for k, s in steps.items())
    steps = OrderedDict((k, remove_not_finite(params[k], s, 0.0)) for k, s in steps.items())
    if tc.get("burn_in_steps", 0):
        remaining = state.setdefault("burn_in", tc["burn_in_steps"])
        mult = 1.0 if remaining <= 0 else 0.0                   # lvsr/algorithms.py:35-43
        steps = OrderedDict((k, s * mult) for k, s in steps.items())
        state["burn_in"] = max(0, remaining - 1)
    return steps


def train_step(cfg, params, state, batch, tc):
    """One GradientDescent.process_batch (B/algorithms/__init__.py:284-287) on float64 parameters.
    batch = (recordings, recordings_mask, labels, labels_mask).  Returns (new_params, cost, grads)."""
    cost, grads = cost_and_grads(cfg, params, *batch, decay=tc.get("decay", 0.0))
    p64 = OrderedDict((k, np.asarray(v, dtype=np.float64)) for k, v in params.items())
    steps = apply_step_rules(p64, grads, state, tc)
    new = OrderedDict((k, p64[k] - steps[k]) for k in p64)
    return new, cost, grads
