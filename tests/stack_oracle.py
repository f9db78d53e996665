"""Float64 oracle of the stacked decoder (net.dec_stack: 2) -- TEST INFRASTRUCTURE ONLY.

With dec_stack 2 the reference's transition is RecurrentStack([GatedRecurrent "transition_0",
GatedRecurrent "transition_1"], skip_connections=True) (lvsr/bricks/recognizer.py:250-259,
libs/blocks/blocks/bricks/recurrent.py:677-968).  Everything else is oracle/lvsr_oracle.py's (and, for content
attention, tests/content_oracle.py's); only what the stack changes is restated here:

  * parameters (Blocks names): the layers are renamed "transition_0#0" / "transition_1#1" under the brick
    "recurrentstack" (its default name) inside att_trans; the stack's fork_1 of layer 0's state has no bias under
    skip connections and is named after layer 1's own sequences (fork_inputs, fork_gate_inputs); every brick that
    took "states" or "inputs" / "gate_inputs" takes "states#1" / "inputs#1" / "gate_inputs#1" too: the attention's
    state_trans, the readout's merge, the generator's fork (with bias) and the distribute fork;
  * transition (recurrent_stack_step): layer 0 is the single-layer GRU step; layer 1's inputs are the distributed
    glimpses + the feedback fork#1 + fork_1 of layer 0's NEW state (recurrent.py:925-950); both take the row mask;
  * attention and readout receive both states and sum one Linear per state (lvsr/bricks/attention.py:103-106,
    the Merge of lvsr/bricks/recognizer.py:298-301).  That sum is [s0 | s1] . [W ; W#1]: wide_params() stacks the
    two weights so the oracle's own take_glimpses / readout run on the wide state rows [s0 | s1].

tests/test_dec_stack_cpu.py pins this module: with layer 1 zero it is the single-layer oracle, its transition is
Blocks' TestRecurrentStack.do_many_steps (skip_connections=True) restated with GRU layers, and its parameter table
is the one of the wsj_jan_wsj13v2 recipe.
"""
from collections import OrderedDict

import numpy as np

from oracle import lvsr_oracle as O
import content_oracle as CO

RS = O._TR + "/recurrentstack"
LAYER = (RS + "/transition_0#0", RS + "/transition_1#1")


def make_config(attention_type="content_and_conv", **kw):
    """O.make_config (or content_oracle's) with dec_stack 2."""
    cfg = CO.make_config(**kw) if attention_type == "content" else O.make_config(**kw)
    cfg["dec_stack"] = 2
    return cfg


def _content(cfg):
    return cfg.get("attention_type") == "content"


def _att(cfg):
    return CO.CONT if _content(cfg) else O._ATT


def param_shapes(cfg):
    """Blocks initialisation order (children depth first): the single-layer table with the stack's parameters where
    their bricks sit -- the transitions then fork_1 in place of the transition (RecurrentStack.children =
    transitions + forks), each "#1" input right after its level-0 sibling (the order of the stack's states and
    sequences)."""
    base = CO.param_shapes(cfg) if _content(cfg) else O.param_shapes(cfg)
    C, Cfb = cfg["dim_dec"], cfg["dim_feedback"]
    g, a = O._GEN, _att(cfg)
    out = OrderedDict()
    for name, shape in base.items():
        if name.startswith(O._TR + "/transition."):
            leaf = name.rsplit(".", 1)[1]
            if leaf == "state_to_state":
                for layer in LAYER:
                    out[layer + ".state_to_state"] = (C, C)
                    out[layer + ".state_to_gates"] = (C, 2 * C)
                    out[layer + ".initial_state"] = (C,)
                out[RS + "/fork_1/fork_inputs.W"] = (C, C)
                out[RS + "/fork_1/fork_gate_inputs.W"] = (C, 2 * C)
            continue
        out[name] = shape
        if name in (g + "/readout/merge/transform_states.W", a + "/state_trans/transform_states.W"):
            out[name.replace("transform_states.W", "transform_states#1.W")] = shape
        elif name == g + "/fork/fork_gate_inputs.W":
            out[g + "/fork/fork_inputs#1.b"] = (C,)
            out[g + "/fork/fork_inputs#1.W"] = (Cfb, C)
            out[g + "/fork/fork_gate_inputs#1.b"] = (2 * C,)
            out[g + "/fork/fork_gate_inputs#1.W"] = (Cfb, 2 * C)
        elif name == O._TR + "/distribute/fork_gate_inputs.W":
            out[O._TR + "/distribute/fork_inputs#1.W"] = shape[:1] + (C,)
            out[O._TR + "/distribute/fork_gate_inputs#1.W"] = shape
    return out


def init_params(cfg, seed=1, weights_std=0.01, initial_state_std=0.001, scale=1.0, dtype=np.float64):
    """O.init_params's scheme (one RandomState walked in brick order) over the stack's table."""
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


def from_single(cfg, single):
    """A stack whose layer 0 holds the single-layer parameters `single` and whose layer 1 and "#1" inputs are zero:
    layer 1's state then stays 0 and the model computes what the single-layer one does."""
    out = OrderedDict()
    for name, shape in param_shapes(cfg).items():
        src = name.replace(LAYER[0], O._TR + "/transition")
        out[name] = np.array(single[src]) if src in single else np.zeros(shape)
    return out


def wide_params(cfg, params):
    """params with the attention's and the readout's state weights replaced by [W ; W#1] [2C, .]: the oracle's
    take_glimpses and readout applied to [s0 | s1] then sum the two Linear outputs as the reference does."""
    p = dict(params)
    for name in (_att(cfg) + "/state_trans/transform_states.W", O._GEN + "/readout/merge/transform_states.W"):
        if name in p:
            p[name] = np.vstack([params[name], params[name.replace("transform_states.W", "transform_states#1.W")]])
    return p


# --------------------------------------------------------------------------
# the stacked transition
# --------------------------------------------------------------------------


def recurrent_stack_step(layers, forks, states, inputs, mask=None):
    """RecurrentStack.do_apply with skip_connections=True for one step (recurrent.py:919-961) of GatedRecurrent
    layers.  layers[l] = dict(state_to_state, state_to_gates); forks[l - 1] = dict(inputs=W, gate_inputs=W), the
    bias-free fork_l of layer l - 1's new state; states[l] [B, C_l]; inputs[l] = (inputs, gate_inputs), layer l's
    own sequences.  Every layer takes the mask.  Returns the new states, layer by layer."""
    out = []
    for l, p in enumerate(layers):
        a, g = inputs[l]
        if l > 0:
            a = a + out[-1].dot(forks[l - 1]["inputs"])
            g = g + out[-1].dot(forks[l - 1]["gate_inputs"])
        out.append(O.gru_step(states[l], a, g, p["state_to_state"], p["state_to_gates"], mask))
    return out


def feedback_fork(cfg, params, outputs):
    """readout.feedback + the generator's fork for both layers: ((inputs, gate_inputs), (inputs#1, gate_inputs#1))."""
    low = O.feedback_fork(cfg, params, outputs)
    if cfg.get("embed_outputs", True):
        fb = params[O._GEN + "/readout/lookupfeedback/lookuptable.W"][outputs]
    else:
        fb = np.eye(cfg["num_phonemes"] + 1, dtype=params[O._GEN + "/fork/fork_inputs.W"].dtype)[outputs]
    high = (O.linear(fb, params[O._GEN + "/fork/fork_inputs#1.W"], params[O._GEN + "/fork/fork_inputs#1.b"]),
            O.linear(fb, params[O._GEN + "/fork/fork_gate_inputs#1.W"], params[O._GEN + "/fork/fork_gate_inputs#1.b"]))
    return low, high


def compute_states(cfg, params, states, fed, weighted_averages, mask=None):
    """AttentionRecurrent.compute_states (B/bricks/attention.py:625-662) around the stack: Distribute adds
    ctx . W to all four sequences, then the stacked step.  states [B, 2C] = [s0 | s1] -> [B, 2C]."""
    C, t = cfg["dim_dec"], O._TR
    wa = weighted_averages
    inputs = []
    for (a, g), sfx in zip(fed, ("", "#1")):
        inputs.append((wa.dot(params[t + "/distribute/fork_inputs%s.W" % sfx]) + a,
                       wa.dot(params[t + "/distribute/fork_gate_inputs%s.W" % sfx]) + g))
    layers = [dict(state_to_state=params[lay + ".state_to_state"], state_to_gates=params[lay + ".state_to_gates"])
              for lay in LAYER]
    forks = [dict(inputs=params[RS + "/fork_1/fork_inputs.W"], gate_inputs=params[RS + "/fork_1/fork_gate_inputs.W"])]
    s0, s1 = recurrent_stack_step(layers, forks, [states[:, :C], states[:, C:]], inputs, mask)
    return np.concatenate([s0, s1], axis=1)


# --------------------------------------------------------------------------
# cost, state functions, search
# --------------------------------------------------------------------------


def _glimpses(cfg, wide, attended, P, attended_mask, weights, step, states):
    f = CO.take_glimpses if _content(cfg) else O.take_glimpses
    return f(cfg, wide, attended, P, attended_mask, weights, step, states)


def initial_states(cfg, params, batch_size, attended):
    h0 = np.concatenate([params[LAYER[0] + ".initial_state"], params[LAYER[1] + ".initial_state"]])
    s0 = np.repeat(h0[None, :], batch_size, 0).astype(attended.dtype)
    glimpses = CO.initial_glimpses if _content(cfg) else O.initial_glimpses
    wa, w, e, step = glimpses(cfg, batch_size, attended)
    return OrderedDict(states=s0, outputs=np.full((batch_size,), cfg["num_phonemes"], dtype=np.int64),
                       weighted_averages=wa, weights=w, energies=e, step=step)


def cost_matrix(cfg, params, attended, attended_mask, labels, labels_mask=None, return_all=False):
    """O.cost_matrix with the stacked transition; states [L, B, 2C] are s_{i-1} of both layers."""
    L, B = labels.shape
    wide = wide_params(cfg, params)
    P = (CO.preprocess if _content(cfg) else O.preprocess)(params, attended)
    low, high = feedback_fork(cfg, params, labels)
    st = initial_states(cfg, params, B, attended)
    s, w, step = st["states"], st["weights"], st["step"]
    states_prev, glimpses, all_w, all_e = [], [], [], []
    for i in range(L):
        states_prev.append(s)
        wa, w, e, step = _glimpses(cfg, wide, attended, P, attended_mask, w, step, s)
        s = compute_states(cfg, params, s, ((low[0][i], low[1][i]), (high[0][i], high[1][i])), wa,
                           None if labels_mask is None else labels_mask[i])
        glimpses.append(wa)
        all_w.append(w)
        all_e.append(e)
    states_prev, ctx = np.stack(states_prev), np.stack(glimpses)
    logp = O.log_softmax(O.readout(cfg, wide, states_prev, ctx))
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
    wide = wide_params(cfg, params)
    wa, _, _, _ = _glimpses(cfg, wide, attended, None, attended_mask, st["weights"], st["step"], st["states"])
    return -O.log_softmax(O.readout(cfg, wide, st["states"], wa))


def next_state_computer(cfg, params, attended, attended_mask, st, outputs):
    wide = wide_params(cfg, params)
    wa, w, e, step = _glimpses(cfg, wide, attended, None, attended_mask, st["weights"], st["step"], st["states"])
    s = compute_states(cfg, params, st["states"], feedback_fork(cfg, params, outputs), wa, None)
    return OrderedDict(states=s, outputs=np.asarray(outputs, dtype=np.int64), weighted_averages=wa, weights=w,
                       energies=e, step=step)


def generate_greedy(cfg, params, attended, attended_mask, n_steps):
    B = attended.shape[1]
    st = initial_states(cfg, params, B, attended)
    outs, costs, states = [], [], []
    for _ in range(n_steps):
        lp = logprobs_computer(cfg, params, attended, attended_mask, st)
        y = lp.argmin(axis=1)
        costs.append(lp[np.arange(B), y])
        st = next_state_computer(cfg, params, attended, attended_mask, st, y)
        outs.append(y)
        states.append(st["states"])
    return np.stack(outs), np.stack(costs), np.stack(states)


def beam_search(cfg, params, recordings, beam_size, **kw):
    """O.beam_search (the reference's BeamSearch.search host logic) over the stacked state functions."""
    computers = dict(initial=lambda att: initial_states(cfg, params, 1, att),
                     logprobs=lambda att, m, st: logprobs_computer(cfg, params, att, m, st),
                     next=lambda att, m, st, y: next_state_computer(cfg, params, att, m, st, y))
    return O.beam_search(cfg, params, recordings, beam_size, computers=computers, **kw)
