"""Float64 oracle of the deep readout (net.post_merge_dims: [d_1, .., d_k], k > 1) -- TEST INFRASTRUCTURE ONLY.

The reference builds the readout's post_merge as (lvsr/bricks/recognizer.py:305-320)

    Bias(d_1) -> act -> MLP([act] * (k-1) + [Identity()], [d_j // pieces for d_j in dims] + [V])

so with p = 1 (a Maxout of more pieces cannot run above depth 1):

    h_0    = act(merge(states, glimpses) + post_merge/bias.b)
    h_j    = act(h_{j-1} . linear_{j-1}.W + linear_{j-1}.b),   j = 1 .. k-1
    logits = h_{k-1} . linear_{k-1}.W + linear_{k-1}.b

Everything else is oracle/lvsr_oracle.py's (O.make_config asserts one post-merge layer, so make_config below
builds the single-layer config and widens its post_merge_dims).  The decoder's recurrence never reads the readout,
so the teacher-forced cost takes the oracle's states and glimpses (O.cost_matrix on parameters whose readout is
depth 1, shallow_params) and applies the deep readout to them.  The torch float64 mirror (cost_and_grads, train_step)
restates G._cost_matrix's loop (content_oracle's for content attention) with the deep readout on top and takes G's
step rules.  relu_kinks screens every Rectifier layer for pre-activations on the derivative's jump, and clear_kinks
moves those units' biases off it.

tests/test_readout_depth_cpu.py pins this module: depth 1 is O.readout, the body is Blocks' MLP restated, known
answers for a 2-layer Tanh and a 3-layer Rectifier readout, both mirrors against numpy and central differences, the
kink screen on a hand-built readout.
"""
from collections import OrderedDict

import numpy as np

from helpers import KINK_EPS
from oracle import lvsr_oracle as O
from oracle import lvsr_oracle_grad as G

PM = O._GEN + "/readout/post_merge"


def linear_name(j):
    return PM + "/mlp/linear_%d" % j


def make_config(post_merge_dims, **kw):
    """O.make_config with a post-merge MLP of len(post_merge_dims) layers."""
    dims = [int(d) for d in post_merge_dims]
    cfg = O.make_config(post_merge_dims=dims[:1], **kw)
    cfg["post_merge_dims"] = dims
    return cfg


def param_shapes(cfg):
    """O.param_shapes with the MLP's Linears in place of linear_0: MLP.children = linear_0 .. linear_{k-1}, each
    initialised b before W (B/bricks/interfaces.py:195-200), as linear_0 of the single-layer table."""
    dims, V, p = cfg["post_merge_dims"], cfg["num_phonemes"], cfg["maxout_pieces"]
    out = OrderedDict()
    for name, shape in O.param_shapes(cfg).items():
        if name.startswith(PM + "/mlp/"):
            continue
        out[name] = shape
        if name == PM + "/bias.b":
            for j in range(len(dims)):
                din = dims[j] // p if j == 0 else dims[j]
                dout = dims[j + 1] if j + 1 < len(dims) else V
                out[linear_name(j) + ".b"] = (dout,)
                out[linear_name(j) + ".W"] = (din, dout)
    return out


def init_params(cfg, seed=1, weights_std=0.01, initial_state_std=0.001, scale=1.0, dtype=np.float64):
    """O.init_params's scheme (one RandomState walked in brick order) over the deep table."""
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


def activation(cfg, x):
    act = cfg["post_merge_activation"]
    if act == "maxout":
        return O.maxout(x, cfg["maxout_pieces"])
    if act == "relu":
        return np.maximum(x, 0)
    if act == "tanh":
        return np.tanh(x)
    assert act == "identity", act
    return x


def bias_name(j):
    """The bias added to the pre-activation of h_j: post_merge/bias.b for h_0, linear_{j-1}.b above it."""
    return PM + "/bias.b" if j == 0 else linear_name(j - 1) + ".b"


def pre_activations(cfg, params, states, weighted_averages):
    """[z_0 .. z_{k-1}] of the readout, h_j = act(z_j)."""
    r = weighted_averages.dot(params[O._GEN + "/readout/merge/transform_weighted_averages.W"])
    if cfg["use_states_for_readout"]:
        r = r + states.dot(params[O._GEN + "/readout/merge/transform_states.W"])
    z = [r + params[PM + "/bias.b"]]
    for j in range(len(cfg["post_merge_dims"]) - 1):
        z.append(O.linear(activation(cfg, z[-1]), params[linear_name(j) + ".W"], params[linear_name(j) + ".b"]))
    return z


def hidden(cfg, params, states, weighted_averages):
    """[h_0 .. h_{k-1}] of the readout."""
    return [activation(cfg, z) for z in pre_activations(cfg, params, states, weighted_averages)]


def readout(cfg, params, states, weighted_averages):
    """Readout.readout with the deep post_merge: the logits [.., V]."""
    k = len(cfg["post_merge_dims"])
    h = hidden(cfg, params, states, weighted_averages)[-1]
    return O.linear(h, params[linear_name(k - 1) + ".W"], params[linear_name(k - 1) + ".b"])


def shallow_params(cfg, params):
    """params with a depth-1 readout (zero linear_0 of O.param_shapes' shape) for the oracle's functions whose
    results the readout does not reach (states, glimpses, alignments)."""
    p = OrderedDict((k, v) for k, v in params.items() if not k.startswith(PM + "/mlp/"))
    shapes = O.param_shapes(cfg)
    for leaf in (".b", ".W"):
        p[linear_name(0) + leaf] = np.zeros(shapes[linear_name(0) + leaf])
    return p


def relu_kinks(cfg, params, states, weighted_averages, live=None, eps=KINK_EPS):
    """(j, step, utterance, unit) of every Rectifier pre-activation z_j of h_0 .. h_{k-1} within eps of 0 on a live row
    (live: [L, B] bool, None for every row).  The derivative jumps at 0, and a float32 forward may land on either side of
    it, which changes that row's backward through the unit.  [] for the other activations."""
    if cfg["post_merge_activation"] != "relu":
        return []
    out = []
    for j, z in enumerate(pre_activations(cfg, params, states, weighted_averages)):
        near = np.abs(z) < eps
        if live is not None:
            near &= np.asarray(live, bool)[..., None]
        out += [(j,) + tuple(int(v) for v in i) for i in np.argwhere(near)]
    return out


def clear_kinks(cfg, params, states, weighted_averages, live=None, eps=KINK_EPS):
    """params with the bias of every unit relu_kinks finds moved off the kink, h_0 first (a move in h_j moves every layer
    above it): by the smallest of +-3 eps, +-4 eps, .. that leaves every live row of the unit at least 2 eps from 0.
    Both sides of a comparison take the result, so the float32 forward and the float64 one take the same side of every
    unit.  Returns (params, [(j, unit, shift)]); asserts that the screen of the result is empty."""
    p = OrderedDict(params)
    moved = []
    for j in range(len(cfg["post_merge_dims"]) if cfg["post_merge_activation"] == "relu" else 0):
        z = pre_activations(cfg, p, states, weighted_averages)[j]
        rows = z.reshape(-1, z.shape[-1]) if live is None else z[np.asarray(live, bool)]
        units = np.flatnonzero((np.abs(rows) < eps).any(axis=0))
        if not units.size:
            continue
        b = np.array(p[bias_name(j)], dtype=np.float64)
        for u in units:
            shift = next(s * n * eps for n in range(3, 1000) for s in (1, -1)
                         if (np.abs(rows[:, u] + s * n * eps) >= 2 * eps).all())
            b[u] += shift
            moved.append((j, int(u), shift))
        p[bias_name(j)] = b.astype(np.asarray(params[bias_name(j)]).dtype)
    assert not relu_kinks(cfg, p, states, weighted_averages, live, eps)
    return p, moved


def cost_matrix(cfg, params, attended, attended_mask, labels, labels_mask=None, return_all=False, emitter="softmax"):
    """O.cost_matrix with the deep readout.  emitter "softmax": -log p(label); "readouts": the logits of every symbol
    [L, B, V] (what RewardRegressionEmitter and shallow fusion take)."""
    r = O.cost_matrix(cfg, shallow_params(cfg, params), attended, attended_mask, labels, labels_mask, return_all=True)
    logits = readout(cfg, params, r["states"], r["weighted_averages"])
    if emitter == "readouts":
        return logits
    costs = -np.take_along_axis(O.log_softmax(logits), labels[..., None], axis=-1)[..., 0]
    if labels_mask is not None:
        costs = costs * labels_mask
    if return_all:
        r["costs"] = costs
        return r
    return costs


def recognizer_cost(cfg, params, recordings, recordings_mask, labels, labels_mask, return_all=False):
    attended, attended_mask = O.encoder(cfg, params, recordings, recordings_mask)
    return cost_matrix(cfg, params, attended, attended_mask, labels, labels_mask, return_all)


def logits_computer(cfg, params, attended, attended_mask, st):
    wa, _, _, _ = O.take_glimpses(cfg, params, attended, None, attended_mask, st["weights"], st["step"], st["states"])
    return readout(cfg, params, st["states"], wa)


def logprobs_computer(cfg, params, attended, attended_mask, st):
    return -O.log_softmax(logits_computer(cfg, params, attended, attended_mask, st))


def next_state_computer(cfg, params, attended, attended_mask, st, outputs):
    return O.next_state_computer(cfg, shallow_params(cfg, params), attended, attended_mask, st, outputs)


def initial_states(cfg, params, batch_size, attended):
    return O.initial_states(cfg, shallow_params(cfg, params), batch_size, attended)


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


def computers(cfg, params):
    return dict(context=lambda x: O.context_computer(cfg, params, x),
                initial=lambda att: initial_states(cfg, params, 1, att),
                logprobs=lambda att, m, st: logprobs_computer(cfg, params, att, m, st),
                next=lambda att, m, st, y: next_state_computer(cfg, params, att, m, st, y))


def beam_search(cfg, params, recordings, beam_size, **kw):
    """O.beam_search (the reference's BeamSearch.search host logic) over the deep readout's state functions."""
    return O.beam_search(cfg, params, recordings, beam_size, computers=computers(cfg, params), **kw)


# --------------------------------------------------------------------------
# torch float64 mirror: gradients and the training step
# --------------------------------------------------------------------------


def _activation_torch(cfg, x):
    import torch
    act = cfg["post_merge_activation"]
    if act == "maxout":
        p = cfg["maxout_pieces"]
        return x.reshape(x.shape[:-1] + (x.shape[-1] // p, p)).max(dim=-1).values
    if act == "relu":
        return torch.clamp(x, min=0)
    if act == "tanh":
        return torch.tanh(x)
    return x


def readout_torch(cfg, p, states, weighted_averages):
    """mirror of readout above."""
    r = weighted_averages @ p[O._GEN + "/readout/merge/transform_weighted_averages.W"]
    if cfg["use_states_for_readout"]:
        r = r + states @ p[O._GEN + "/readout/merge/transform_states.W"]
    h = _activation_torch(cfg, r + p[PM + "/bias.b"])
    k = len(cfg["post_merge_dims"])
    for j in range(k - 1):
        h = _activation_torch(cfg, h @ p[linear_name(j) + ".W"] + p[linear_name(j) + ".b"])
    return h @ p[linear_name(k - 1) + ".W"] + p[linear_name(k - 1) + ".b"]


def _cost_matrix_torch(cfg, p, attended, attended_mask, labels, labels_mask):
    """mirror of cost_matrix above: G._cost_matrix's teacher-forced loop, then the deep readout."""
    import torch
    L, B = labels.shape
    P = attended @ p[O._ATT + "/preprocess.W"] + p[O._ATT + "/preprocess.b"]
    if cfg.get("embed_outputs", True):
        fb = p[O._GEN + "/readout/lookupfeedback/lookuptable.W"][torch.as_tensor(labels)]
    else:
        fb = torch.eye(cfg["num_phonemes"] + 1, dtype=attended.dtype)[torch.as_tensor(labels)]
    inputs = fb @ p[O._GEN + "/fork/fork_inputs.W"] + p[O._GEN + "/fork/fork_inputs.b"]
    gate_inputs = fb @ p[O._GEN + "/fork/fork_gate_inputs.W"] + p[O._GEN + "/fork/fork_gate_inputs.b"]
    s = p[O._TR + "/transition.initial_state"][None, :].expand(B, -1)
    w = torch.zeros((B, attended.shape[0]), dtype=attended.dtype)
    w[:, 0] = 1
    step = np.zeros((B,), dtype=np.int64)
    prev, ctxs = [], []
    for i in range(L):
        prev.append(s)
        wavg, w, step = G._take_glimpses(cfg, p, attended, P, attended_mask, w, step, s)
        a = wavg @ p[O._TR + "/distribute/fork_inputs.W"] + inputs[i]
        g = wavg @ p[O._TR + "/distribute/fork_gate_inputs.W"] + gate_inputs[i]
        s = G._gru_step(s, a, g, p[O._TR + "/transition.state_to_state"], p[O._TR + "/transition.state_to_gates"],
                        None if labels_mask is None else labels_mask[i])
        ctxs.append(wavg)
    logp = torch.log_softmax(readout_torch(cfg, p, torch.stack(prev), torch.stack(ctxs)), dim=-1)
    costs = -torch.gather(logp, 2, torch.as_tensor(labels)[..., None])[..., 0]
    if labels_mask is not None:
        costs = costs * labels_mask
    return costs


def _content_cost_matrix_torch(cfg, p, attended, attended_mask, labels, labels_mask):
    """mirror of cost_matrix above over content attention (attention_type: content): content_oracle's loop, then the
    deep readout."""
    import content_oracle as CO
    return CO._cost_matrix_torch(cfg, p, attended, attended_mask, labels, labels_mask, readout=readout_torch)


def cost_and_grads(cfg, params, recordings, recordings_mask, labels, labels_mask, decay=0.0, return_costs=False):
    """G.cost_and_grads for the deep readout: sum(costs) / B (+ decay * ||WEIGHT||^2) and its float64 gradient.  A
    content-attention config (content_oracle.make_config) runs the content mirror."""
    import torch
    p = OrderedDict((k, torch.tensor(np.asarray(v, dtype=np.float64), requires_grad=True)) for k, v in params.items())
    x = torch.as_tensor(np.asarray(recordings, dtype=np.float64))
    m = None if recordings_mask is None else torch.as_tensor(np.asarray(recordings_mask, dtype=np.float64))
    lm = None if labels_mask is None else torch.as_tensor(np.asarray(labels_mask, dtype=np.float64))
    labels = np.asarray(labels, dtype=np.int64)
    attended, amask = G._encoder(cfg, p, x, m)
    mirror = _content_cost_matrix_torch if cfg.get("attention_type") == "content" else _cost_matrix_torch
    costs = mirror(cfg, p, attended, amask, labels, lm)
    cost = costs.sum() / labels.shape[1]
    if decay > 0:
        cost = cost + decay * sum((v ** 2).sum() for k, v in p.items() if G.is_weight(k))
    grads = torch.autograd.grad(cost, list(p.values()), allow_unused=True)
    out = OrderedDict((k, np.zeros(v.shape) if g is None else g.numpy().copy()) for (k, v), g in zip(p.items(), grads))
    if return_costs:
        return float(cost.detach()), out, costs.detach().numpy()
    return float(cost.detach()), out


def train_step(cfg, params, state, batch, tc):
    """G.train_step for the deep readout: gradients, then the oracle's step rules."""
    cost, grads = cost_and_grads(cfg, params, *batch, decay=tc.get("decay", 0.0))
    p64 = OrderedDict((k, np.asarray(v, dtype=np.float64)) for k, v in params.items())
    steps = G.apply_step_rules(p64, grads, state, tc)
    return OrderedDict((k, p64[k] - steps[k]) for k in p64), cost, grads
