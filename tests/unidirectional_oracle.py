"""Float64 oracle of the unidirectional encoder (net.bidir: False) -- TEST INFRASTRUCTURE ONLY.

With bidir False the reference's Encoder (lvsr/bricks/__init__.py:54-78) does not wrap its layers in Bidirectional:
layer l is RecurrentWithFork(GatedRecurrent(dim=D_l), name="with_fork<l>") scanned forward from its initial state,
layer l > 0 takes D_{l-1} features (dims_under = [dim_input] + dims) and the encoded width is dims[-1].  Everything
after the encoder is oracle/lvsr_oracle.py's (tests/content_oracle.py's for content attention) at E = dims[-1]; only
what the flag changes is restated here:

  * parameters (Blocks names): "/recognizer/encoder/with_fork<l>/gatedrecurrent.{state_to_state, state_to_gates,
    initial_state}" then "/recognizer/encoder/with_fork<l>/fork/fork_{inputs, gate_inputs}.{b, W}"
    (RecurrentWithFork.children = [recurrent.brick, fork]), in place of each layer's two Bidirectional children;
  * encoder: O.recurrent_with_fork(..., reverse=False) per layer, then x[::k] as before;
  * the decoder functions take decoder_config(cfg), the same config with the one-layer bidirectional encoder
    [E / 2] whose encoded width is E: they read the encoder's width only through O.dim_encoded.

tests/test_unidirectional_cpu.py pins this module: one layer equals the forward half of O.bidirectional with the
same parameters, the torch mirror equals numpy, autograd agrees with finite differences, and the parameter table is a
hand-written Blocks list.
"""
from collections import OrderedDict

import numpy as np

from oracle import lvsr_oracle as O
from oracle import lvsr_oracle_grad as G
import content_oracle as CO

ENC = "/recognizer/encoder"


def make_config(attention_type="content_and_conv", **kw):
    """O.make_config (or content_oracle's) with bidir False."""
    cfg = CO.make_config(**kw) if attention_type == "content" else O.make_config(**kw)
    cfg["bidir"] = False
    return cfg


def _content(cfg):
    return cfg.get("attention_type") == "content"


def layer_base(l):
    return "%s/with_fork%d" % (ENC, l)


def dim_encoded(cfg):
    return cfg["dims_bidir"][-1]


def decoder_config(cfg):
    """cfg as the decoder functions of O / CO read it: their only view of the encoder is O.dim_encoded = E."""
    E = dim_encoded(cfg)
    assert E % 2 == 0
    out = dict(cfg)
    out["dims_bidir"] = [E // 2]
    out["subsample"] = [1]
    out.pop("bidir", None)
    return out


def param_shapes(cfg):
    """Blocks initialisation order: the forward-only encoder layers, then the decoder's table at E = dims[-1]."""
    shapes = OrderedDict()
    din = cfg["num_features"]
    for l, D in enumerate(cfg["dims_bidir"]):
        base = layer_base(l)
        shapes[base + "/gatedrecurrent.state_to_state"] = (D, D)
        shapes[base + "/gatedrecurrent.state_to_gates"] = (D, 2 * D)
        shapes[base + "/gatedrecurrent.initial_state"] = (D,)
        shapes[base + "/fork/fork_inputs.b"] = (D,)
        shapes[base + "/fork/fork_inputs.W"] = (din, D)
        shapes[base + "/fork/fork_gate_inputs.b"] = (2 * D,)
        shapes[base + "/fork/fork_gate_inputs.W"] = (din, 2 * D)
        din = D
    dcfg = decoder_config(cfg)
    dec = CO.param_shapes(dcfg) if _content(cfg) else O.param_shapes(dcfg)
    for name, shape in dec.items():
        if not name.startswith(ENC + "/"):
            shapes[name] = shape
    return shapes


def init_params(cfg, seed=1, weights_std=0.01, initial_state_std=0.001, scale=1.0, dtype=np.float64):
    """O.init_params's scheme (one RandomState walked in brick order) over the unidirectional table."""
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


def encoder(cfg, params, x, mask=None, return_layers=False):
    """lvsr/bricks/__init__.py:71-78 with bidir False: x [T,B,F], mask [T,B] -> (encoded [T',B,E], encoded_mask)."""
    layers = []
    for l, k in enumerate(cfg["subsample"]):
        x = O.recurrent_with_fork(x, mask, params, layer_base(l), reverse=False)[::k]
        if mask is not None:
            mask = mask[::k]
        layers.append(x)
    enc_mask = mask if mask is not None else np.ones_like(x[:, :, 0])
    if return_layers:
        return x, enc_mask, layers
    return x, enc_mask


def _dec(cfg):
    return CO if _content(cfg) else O


def cost_matrix(cfg, params, attended, attended_mask, labels, labels_mask=None, return_all=False):
    return _dec(cfg).cost_matrix(decoder_config(cfg), params, attended, attended_mask, labels, labels_mask, return_all)


def recognizer_cost(cfg, params, recordings, recordings_mask, labels, labels_mask, return_all=False):
    attended, attended_mask = encoder(cfg, params, recordings, recordings_mask)
    return cost_matrix(cfg, params, attended, attended_mask, labels, labels_mask, return_all)


def initial_states(cfg, params, batch_size, attended):
    return _dec(cfg).initial_states(decoder_config(cfg), params, batch_size, attended)


def logprobs_computer(cfg, params, attended, attended_mask, st):
    return _dec(cfg).logprobs_computer(decoder_config(cfg), params, attended, attended_mask, st)


def next_state_computer(cfg, params, attended, attended_mask, st, outputs):
    return _dec(cfg).next_state_computer(decoder_config(cfg), params, attended, attended_mask, st, outputs)


def generate_greedy(cfg, params, attended, attended_mask, n_steps):
    return _dec(cfg).generate_greedy(decoder_config(cfg), params, attended, attended_mask, n_steps)


def beam_search(cfg, params, recordings, beam_size, **kw):
    """O.beam_search (the reference's BeamSearch.search host logic) over the unidirectional context and the state
    functions above (search runs the encoder unmasked, lvsr/bricks/recognizer.py:503)."""
    computers = dict(context=lambda x: encoder(cfg, params, x, None),
                     initial=lambda att: initial_states(cfg, params, 1, att),
                     logprobs=lambda att, m, st: logprobs_computer(cfg, params, att, m, st),
                     next=lambda att, m, st, y: next_state_computer(cfg, params, att, m, st, y))
    return O.beam_search(decoder_config(cfg), params, recordings, beam_size, computers=computers, **kw)


# --------------------------------------------------------------------------
# torch float64 mirror (gradients), from lvsr_oracle_grad's pieces
# --------------------------------------------------------------------------


def _encoder_torch(cfg, p, x, mask):
    """mirror of encoder above in the style of G._encoder."""
    import torch
    for l, k in enumerate(cfg["subsample"]):
        base = layer_base(l)
        a = x @ p[base + "/fork/fork_inputs.W"] + p[base + "/fork/fork_inputs.b"]
        g = x @ p[base + "/fork/fork_gate_inputs.W"] + p[base + "/fork/fork_gate_inputs.b"]
        h = p[base + "/gatedrecurrent.initial_state"][None, :].expand(x.shape[1], -1)
        seq = []
        for t in range(x.shape[0]):
            h = G._gru_step(h, a[t], g[t], p[base + "/gatedrecurrent.state_to_state"],
                            p[base + "/gatedrecurrent.state_to_gates"], None if mask is None else mask[t])
            seq.append(h)
        x = torch.stack(seq)[::k]
        if mask is not None:
            mask = mask[::k]
    return x, (mask if mask is not None else torch.ones_like(x[:, :, 0]))


def cost_and_grads(cfg, params, recordings, recordings_mask, labels, labels_mask, decay=0.0, return_costs=False):
    """G.cost_and_grads for the unidirectional model: sum(costs) / B (+ decay * ||WEIGHT||^2), float64 gradients."""
    import torch
    p = OrderedDict((k, torch.tensor(np.asarray(v, dtype=np.float64), requires_grad=True)) for k, v in params.items())
    x = torch.as_tensor(np.asarray(recordings, dtype=np.float64))
    m = None if recordings_mask is None else torch.as_tensor(np.asarray(recordings_mask, dtype=np.float64))
    lm = None if labels_mask is None else torch.as_tensor(np.asarray(labels_mask, dtype=np.float64))
    labels = np.asarray(labels, dtype=np.int64)
    attended, amask = _encoder_torch(cfg, p, x, m)
    dcfg = decoder_config(cfg)
    if _content(cfg):
        costs = CO._cost_matrix_torch(dcfg, p, attended, amask, labels, lm)
    else:
        costs = G._cost_matrix(dcfg, p, attended, amask, labels, lm)
    cost = costs.sum() / labels.shape[1]
    if decay > 0:
        cost = cost + decay * sum((v ** 2).sum() for k, v in p.items() if G.is_weight(k))
    grads = torch.autograd.grad(cost, list(p.values()), allow_unused=True)
    out = OrderedDict((k, np.zeros(v.shape) if g is None else g.numpy().copy()) for (k, v), g in zip(p.items(), grads))
    if return_costs:
        return float(cost.detach()), out, costs.detach().numpy()
    return float(cost.detach()), out


def train_step(cfg, params, state, batch, tc):
    """G.train_step for the unidirectional model: gradients, then the oracle's step rules."""
    cost, grads = cost_and_grads(cfg, params, *batch, decay=tc.get("decay", 0.0))
    p64 = OrderedDict((k, np.asarray(v, dtype=np.float64)) for k, v in params.items())
    steps = G.apply_step_rules(p64, grads, state, tc)
    return OrderedDict((k, p64[k] - steps[k]) for k in p64), cost, grads
