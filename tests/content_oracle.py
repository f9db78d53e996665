"""Float64 oracle of content-only attention (attention_type: content) -- TEST INFRASTRUCTURE ONLY.

SequenceContentAttention ("cont_att", libs/blocks/blocks/bricks/attention.py:259-414; built by
lvsr/bricks/recognizer.py:261-265) inside the same recognizer as oracle/lvsr_oracle.py, which models the
content_and_conv mechanism.  Everything that does not depend on the attention (encoder, feedback, transition,
readout, the BeamSearch host logic, the step rules) is the oracle's own code; only the attention and what
calls it are restated here:

  * parameters: state_trans/transform_states.W [C,M], preprocess.b [M], preprocess.W [E,M],
    energy_comp/linear.W [M,1] in place of the conv_att block (no handler, filters or energy bias);
  * take_glimpses: e = tanh(P + s.W_s).v over every frame, softmax weights by the generic compute_weights
    (max over masked positions too, +1 when a column is fully masked), weighted average;
  * initial glimpses: zeros, weights included (:392-395); no energies state, so energies are zeros
    (what analyze reports, lvsr/bricks/recognizer.py:475-478);
  * conv_n, conv_num_filters, energy_normalizer and prior are not passed to this brick: they are ignored.

The torch float64 mirror (cost_and_grads, train_step) reuses oracle/lvsr_oracle_grad.py's encoder, GRU step,
weights and step rules.  tests/test_content_attention_cpu.py pins this module: the reference's frozen attention
sums 113.429 / 415.901 through take_glimpses, the mirror against the numpy functions, autograd against finite
differences.
"""
from collections import OrderedDict

import numpy as np

from oracle import lvsr_oracle as O
from oracle import lvsr_oracle_grad as G

CONT = "/recognizer/generator/att_trans/cont_att"
_IGNORED = ("attention_type", "energy_normalizer", "prior")


def make_config(**kw):
    """O.make_config for a content-attention recognizer; the keys the brick does not take are dropped."""
    cfg = O.make_config(**{k: v for k, v in kw.items() if k not in _IGNORED})
    cfg["attention_type"] = "content"
    return cfg


def param_shapes(cfg):
    """Blocks order: the content_and_conv table with the conv_att block replaced by cont_att's children
    [state_trans, preprocess, energy_comp] (B/bricks/attention.py:361-368)."""
    C, M, E = cfg["dim_dec"], cfg["dim_matcher"], O.dim_encoded(cfg)
    out = OrderedDict()
    for name, shape in O.param_shapes(cfg).items():
        if O._ATT not in name:
            out[name] = shape
        elif name.endswith("/state_trans/transform_states.W"):
            out[CONT + "/state_trans/transform_states.W"] = (C, M)
            out[CONT + "/preprocess.b"] = (M,)
            out[CONT + "/preprocess.W"] = (E, M)
            out[CONT + "/energy_comp/linear.W"] = (M, 1)
    return out


def init_params(cfg, seed=1, weights_std=0.01, initial_state_std=0.001, scale=1.0, dtype=np.float64):
    """O.init_params's scheme (one RandomState walked in brick order) over the content parameter table."""
    rng = np.random.RandomState(seed)
    out = OrderedDict()
    for name, shape in param_shapes(cfg).items():
        leaf = name.rsplit(".", 1)[1]
        if leaf == "b":
            v = np.zeros(shape)
        elif leaf == "state_to_state":
            v = O.orthogonal(rng, shape)
        elif leaf == "state_to_gates":
            D = shape[0]
            v = np.hstack([O.orthogonal(rng, (D, D)), O.orthogonal(rng, (D, D))])
        elif leaf == "initial_state":
            v = rng.normal(0, initial_state_std, size=shape) * scale
        else:
            v = rng.normal(0, weights_std, size=shape) * scale
        out[name] = np.ascontiguousarray(v, dtype=dtype)
    return out


def preprocess(params, attended):
    """B/bricks/attention.py:405-414."""
    return O.linear(attended, params[CONT + "/preprocess.W"], params[CONT + "/preprocess.b"])


def take_glimpses(cfg, params, attended, preprocessed, attended_mask, weights, step, states):
    """SequenceContentAttention.take_glimpses (B/bricks/attention.py:370-388), with the state layout of
    O.take_glimpses: -> weighted_averages [B,E], weights [B,T'], energies (zeros) [B,T'], step + 1 (only counted)."""
    if preprocessed is None:
        preprocessed = preprocess(params, attended)
    wa, w = O.content_take_glimpses(attended, preprocessed, attended_mask, states,
                                    params[CONT + "/state_trans/transform_states.W"],
                                    params[CONT + "/energy_comp/linear.W"])
    return wa, w, np.zeros_like(w), step + 1


def initial_glimpses(cfg, batch_size, attended):
    """B/bricks/attention.py:392-395: zero weighted averages AND weights; zero energies, step 0."""
    z = np.zeros((batch_size, attended.shape[0]), dtype=attended.dtype)
    return (np.zeros((batch_size, O.dim_encoded(cfg)), dtype=attended.dtype), z.copy(), z.copy(),
            np.zeros((batch_size,), dtype=np.int64))


def initial_states(cfg, params, batch_size, attended):
    s0 = np.repeat(params[O._TR + "/transition.initial_state"][None, :], batch_size, 0).astype(attended.dtype)
    wa, w, e, step = initial_glimpses(cfg, batch_size, attended)
    return OrderedDict(states=s0, outputs=np.full((batch_size,), cfg["num_phonemes"], dtype=np.int64),
                       weighted_averages=wa, weights=w, energies=e, step=step)


def cost_matrix(cfg, params, attended, attended_mask, labels, labels_mask=None, return_all=False):
    """O.cost_matrix with the content attention (B/bricks/sequence_generators.py:254-326)."""
    L, B = labels.shape
    P = preprocess(params, attended)
    inputs, gate_inputs = O.feedback_fork(cfg, params, labels)
    st = initial_states(cfg, params, B, attended)
    s, w, step = st["states"], st["weights"], st["step"]
    states_prev, glimpses, all_w, all_e = [], [], [], []
    for i in range(L):
        states_prev.append(s)
        wa, w, e, step = take_glimpses(cfg, params, attended, P, attended_mask, w, step, s)
        s = O.compute_states(cfg, params, s, inputs[i], gate_inputs[i], wa,
                             None if labels_mask is None else labels_mask[i])
        glimpses.append(wa)
        all_w.append(w)
        all_e.append(e)
    states_prev, ctx = np.stack(states_prev), np.stack(glimpses)
    logp = O.log_softmax(O.readout(cfg, params, states_prev, ctx))
    costs = -np.take_along_axis(logp, labels[..., None], axis=-1)[..., 0]
    if labels_mask is not None:
        costs = costs * labels_mask
    if return_all:
        return dict(costs=costs, states=states_prev, weighted_averages=ctx, weights=np.stack(all_w),
                    energies=np.stack(all_e), final_state=s)
    return costs


def recognizer_cost(cfg, params, recordings, recordings_mask, labels, labels_mask, return_all=False):
    attended, attended_mask = O.encoder(cfg, params, recordings, recordings_mask)
    return cost_matrix(cfg, params, attended, attended_mask, labels, labels_mask, return_all)


def logprobs_computer(cfg, params, attended, attended_mask, st):
    wa, _, _, _ = take_glimpses(cfg, params, attended, None, attended_mask, st["weights"], st["step"], st["states"])
    return -O.log_softmax(O.readout(cfg, params, st["states"], wa))


def next_state_computer(cfg, params, attended, attended_mask, st, outputs):
    wa, w, e, step = take_glimpses(cfg, params, attended, None, attended_mask, st["weights"], st["step"], st["states"])
    inputs, gate_inputs = O.feedback_fork(cfg, params, outputs)
    s = O.compute_states(cfg, params, st["states"], inputs, gate_inputs, wa, None)
    return OrderedDict(states=s, outputs=np.asarray(outputs, dtype=np.int64), weighted_averages=wa, weights=w,
                       energies=e, step=step)


def generate_greedy(cfg, params, attended, attended_mask, n_steps):
    B = attended.shape[1]
    st = initial_states(cfg, params, B, attended)
    outs, costs = [], []
    for _ in range(n_steps):
        lp = logprobs_computer(cfg, params, attended, attended_mask, st)
        y = lp.argmin(axis=1)
        costs.append(lp[np.arange(B), y])
        st = next_state_computer(cfg, params, attended, attended_mask, st, y)
        outs.append(y)
    return np.stack(outs), np.stack(costs), st


def beam_search(cfg, params, recordings, beam_size, **kw):
    """O.beam_search (the reference's BeamSearch.search host logic) over the content state functions."""
    computers = dict(initial=lambda att: initial_states(cfg, params, 1, att),
                     logprobs=lambda att, m, st: logprobs_computer(cfg, params, att, m, st),
                     next=lambda att, m, st, y: next_state_computer(cfg, params, att, m, st, y))
    return O.beam_search(cfg, params, recordings, beam_size, computers=computers, **kw)


# --------------------------------------------------------------------------
# torch float64 mirror (gradients)
# --------------------------------------------------------------------------


def _readout_torch(cfg, p, states, weighted_averages):
    """mirror of O.readout: the single-layer post_merge."""
    import torch
    r = weighted_averages @ p[O._GEN + "/readout/merge/transform_weighted_averages.W"]
    if cfg["use_states_for_readout"]:
        r = r + states @ p[O._GEN + "/readout/merge/transform_states.W"]
    r = r + p[O._GEN + "/readout/post_merge/bias.b"]
    act = cfg["post_merge_activation"]
    if act == "maxout":
        pieces = cfg["maxout_pieces"]
        r = r.reshape(r.shape[:-1] + (r.shape[-1] // pieces, pieces)).max(dim=-1).values
    elif act == "relu":
        r = torch.clamp(r, min=0)
    elif act == "tanh":
        r = torch.tanh(r)
    return r @ p[O._GEN + "/readout/post_merge/mlp/linear_0.W"] + p[O._GEN + "/readout/post_merge/mlp/linear_0.b"]


def _cost_matrix_torch(cfg, p, attended, attended_mask, labels, labels_mask, readout=_readout_torch):
    """mirror of cost_matrix above, in the style of G._cost_matrix; `readout(cfg, p, states, weighted_averages)` gives
    the logits of every step (readout_oracle.readout_torch for a deep readout)."""
    import torch
    L, B = labels.shape
    P = attended @ p[CONT + "/preprocess.W"] + p[CONT + "/preprocess.b"]
    if cfg.get("embed_outputs", True):
        fb = p[O._GEN + "/readout/lookupfeedback/lookuptable.W"][torch.as_tensor(labels)]
    else:
        fb = torch.eye(cfg["num_phonemes"] + 1, dtype=attended.dtype)[torch.as_tensor(labels)]
    inputs = fb @ p[O._GEN + "/fork/fork_inputs.W"] + p[O._GEN + "/fork/fork_inputs.b"]
    gate_inputs = fb @ p[O._GEN + "/fork/fork_gate_inputs.W"] + p[O._GEN + "/fork/fork_gate_inputs.b"]
    s = p[O._TR + "/transition.initial_state"][None, :].expand(B, -1)
    prev, ctxs = [], []
    for i in range(L):
        prev.append(s)
        match = P + (s @ p[CONT + "/state_trans/transform_states.W"])[None]
        e = (torch.tanh(match) @ p[CONT + "/energy_comp/linear.W"])[..., 0]
        w = G._compute_weights(e, attended_mask, "softmax")
        wavg = (w[:, :, None] * attended).sum(dim=0)
        a = wavg @ p[O._TR + "/distribute/fork_inputs.W"] + inputs[i]
        g = wavg @ p[O._TR + "/distribute/fork_gate_inputs.W"] + gate_inputs[i]
        s = G._gru_step(s, a, g, p[O._TR + "/transition.state_to_state"], p[O._TR + "/transition.state_to_gates"],
                        None if labels_mask is None else labels_mask[i])
        ctxs.append(wavg)
    logp = torch.log_softmax(readout(cfg, p, torch.stack(prev), torch.stack(ctxs)), dim=-1)
    costs = -torch.gather(logp, 2, torch.as_tensor(labels)[..., None])[..., 0]
    if labels_mask is not None:
        costs = costs * labels_mask
    return costs


def cost_and_grads(cfg, params, recordings, recordings_mask, labels, labels_mask, decay=0.0, return_costs=False):
    """G.cost_and_grads for the content model: sum(costs) / B (+ decay * ||WEIGHT||^2) and its float64 gradient."""
    import torch
    p = OrderedDict((k, torch.tensor(np.asarray(v, dtype=np.float64), requires_grad=True)) for k, v in params.items())
    x = torch.as_tensor(np.asarray(recordings, dtype=np.float64))
    m = None if recordings_mask is None else torch.as_tensor(np.asarray(recordings_mask, dtype=np.float64))
    lm = None if labels_mask is None else torch.as_tensor(np.asarray(labels_mask, dtype=np.float64))
    labels = np.asarray(labels, dtype=np.int64)
    attended, amask = G._encoder(cfg, p, x, m)
    costs = _cost_matrix_torch(cfg, p, attended, amask, labels, lm)
    cost = costs.sum() / labels.shape[1]
    if decay > 0:
        cost = cost + decay * sum((v ** 2).sum() for k, v in p.items() if G.is_weight(k))
    grads = torch.autograd.grad(cost, list(p.values()), allow_unused=True)
    out = OrderedDict((k, np.zeros(v.shape) if g is None else g.numpy().copy()) for (k, v), g in zip(p.items(), grads))
    if return_costs:
        return float(cost.detach()), out, costs.detach().numpy()
    return float(cost.detach()), out


def train_step(cfg, params, state, batch, tc):
    """G.train_step for the content model: gradients, then the oracle's step rules."""
    cost, grads = cost_and_grads(cfg, params, *batch, decay=tc.get("decay", 0.0))
    p64 = OrderedDict((k, np.asarray(v, dtype=np.float64)) for k, v in params.items())
    steps = G.apply_step_rules(p64, grads, state, tc)
    return OrderedDict((k, p64[k] - steps[k]) for k in p64), cost, grads
