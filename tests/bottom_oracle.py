"""Float64 oracle of the bottom MLP (net.bottom.dims non-empty) -- TEST INFRASTRUCTURE ONLY.

SpeechBottom (lvsr/bricks/recognizer.py:105-157) with dims = [d1, ..., dk] is Blocks' MLP([act] * k,
[num_features] + dims, name="bottom") applied to every frame of the recordings, before the encoder
(:378-400): x_{i+1} = act(x_i W_i + b_i).  The activation is Rectifier (switch(x > 0, x, 0), so its derivative at 0
is 0) or Tanh, which is what None means (:116-117).  The bottom is a pure function of the recordings, so the model
behind it is the oracle's own model with num_features = dk (inner()); only the bottom and its place in the parameter
table are restated here:

  * parameters: /recognizer/bottom/bottom/linear_<i>.W [d_in, d_out] then .b [d_out] (MLP names its linears
    linear_<i>, libs/blocks/blocks/bricks/sequences.py:119-123; Linear._allocate makes W first), after the encoder's
    and before the generator's (SpeechRecognizer.children = [encoder, top, bottom, generator], :350);
  * every entry point starting from recordings runs the inner model's on bottom(recordings): lvsr_oracle for
    content_and_conv attention, content_oracle for content attention, stack_oracle for dec_stack 2;
  * the torch float64 mirror (cost_and_grads, train_step) puts the bottom in front of lvsr_oracle_grad's encoder;
  * a forward-only encoder (cfg["bidir"] False, unidirectional_oracle.make_config's configs) takes
    unidirectional_oracle's table, encoder and decoder functions in place of lvsr_oracle's.

tests/test_bottom_cpu.py pins this module: Blocks' test_mlp known answer, the Rectifier at 0, the mirror against the
numpy functions, autograd against finite differences.
"""
from collections import OrderedDict

import numpy as np

from oracle import lvsr_oracle as O
from oracle import lvsr_oracle_grad as G
import content_oracle as CO
import stack_oracle as SO
import unidirectional_oracle as U

BOTTOM = "/recognizer/bottom/bottom"


def make_config(cfg, dims, activation="relu"):
    """`cfg` (a config of lvsr_oracle, content_oracle or stack_oracle) with the bottom MLP `dims`; activation
    "relu" (Rectifier) or "tanh" (None means Tanh)."""
    out = dict(cfg)
    out["bottom"] = dict(dims=[int(d) for d in dims], activation=activation or "tanh")
    return out


def inner(cfg):
    """The config of the model behind the bottom: the same with num_features = the bottom's last width."""
    out = {k: v for k, v in cfg.items() if k != "bottom"}
    if cfg.get("bottom") and cfg["bottom"]["dims"]:
        out["num_features"] = cfg["bottom"]["dims"][-1]
    return out


def _unidirectional(cfg):
    return cfg.get("bidir", True) is False


def _module(cfg):
    if _unidirectional(cfg):
        return U
    if cfg.get("dec_stack", 1) == 2:
        return SO
    return CO if cfg.get("attention_type") == "content" else O


def linear_name(i):
    return "%s/linear_%d" % (BOTTOM, i)


def param_shapes(cfg):
    """The inner model's table with the bottom's parameters after the encoder's."""
    base = _module(cfg).param_shapes(inner(cfg))
    out = OrderedDict()
    placed = False
    for name, shape in base.items():
        if not placed and not name.startswith("/recognizer/encoder/"):
            din = cfg["num_features"]
            for i, d in enumerate(cfg.get("bottom", {}).get("dims", [])):
                out[linear_name(i) + ".W"] = (din, d)
                out[linear_name(i) + ".b"] = (d,)
                din = d
            placed = True
        out[name] = shape
    return out


def init_params(cfg, seed=1, weights_std=0.01, initial_state_std=0.001, scale=1.0, dtype=np.float64):
    """O.init_params's scheme (one RandomState walked in brick order) over the table with the bottom."""
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


def rectifier(x):
    """blocks.bricks.Rectifier: switch(x > 0, x, 0)."""
    return np.where(x > 0, x, 0.0)


ACTIVATIONS = {"relu": rectifier, "tanh": np.tanh}


def pre_activations(cfg, params, x):
    """[x_i W_i + b_i for every layer i] on frames x [..., F]."""
    out = []
    act = ACTIVATIONS[cfg["bottom"]["activation"]]
    for i in range(len(cfg["bottom"]["dims"])):
        z = O.linear(x, params[linear_name(i) + ".W"], params[linear_name(i) + ".b"])
        out.append(z)
        x = act(z)
    return out


def bottom(cfg, params, x):
    """SpeechBottom.apply: the MLP on every frame of x [..., F] -> [..., dk]; x itself without a bottom."""
    if not cfg.get("bottom") or not cfg["bottom"]["dims"]:
        return x
    return ACTIVATIONS[cfg["bottom"]["activation"]](pre_activations(cfg, params, x)[-1])


def encoder(cfg, params, x, mask=None):
    return (U if _unidirectional(cfg) else O).encoder(inner(cfg), params, bottom(cfg, params, x), mask)


def recognizer_cost(cfg, params, recordings, recordings_mask, labels, labels_mask, return_all=False):
    return _module(cfg).recognizer_cost(inner(cfg), params, bottom(cfg, params, recordings), recordings_mask, labels,
                                        labels_mask, return_all)


def generate_greedy(cfg, params, recordings, recordings_mask, n_steps):
    attended, attended_mask = encoder(cfg, params, recordings, recordings_mask)
    return _module(cfg).generate_greedy(inner(cfg), params, attended, attended_mask, n_steps)


def beam_search(cfg, params, recordings, beam_size, **kw):
    """The inner model's beam search on bottom(recordings [T, F]); max_length still follows T."""
    return _module(cfg).beam_search(inner(cfg), params, bottom(cfg, params, recordings), beam_size, **kw)


# --------------------------------------------------------------------------
# torch float64 mirror (gradients)
# --------------------------------------------------------------------------


def _bottom_torch(cfg, p, x):
    import torch
    if not cfg.get("bottom") or not cfg["bottom"]["dims"]:
        return x
    for i in range(len(cfg["bottom"]["dims"])):
        z = x @ p[linear_name(i) + ".W"] + p[linear_name(i) + ".b"]
        # Rectifier's gradient is switch(z > 0, 1, 0): 0 at z = 0, as Theano's
        x = torch.where(z > 0, z, torch.zeros_like(z)) if cfg["bottom"]["activation"] == "relu" else torch.tanh(z)
    return x


def cost_and_grads(cfg, params, recordings, recordings_mask, labels, labels_mask, decay=0.0, return_costs=False):
    """G.cost_and_grads with the bottom: sum(costs) / B (+ decay * ||WEIGHT||^2) and its float64 gradient."""
    import torch
    p = OrderedDict((k, torch.tensor(np.asarray(v, dtype=np.float64), requires_grad=True)) for k, v in params.items())
    x = torch.as_tensor(np.asarray(recordings, dtype=np.float64))
    m = None if recordings_mask is None else torch.as_tensor(np.asarray(recordings_mask, dtype=np.float64))
    lm = None if labels_mask is None else torch.as_tensor(np.asarray(labels_mask, dtype=np.float64))
    labels = np.asarray(labels, dtype=np.int64)
    icfg = inner(cfg)
    if _unidirectional(cfg):
        attended, amask = U._encoder_torch(icfg, p, _bottom_torch(cfg, p, x), m)
        icfg = U.decoder_config(icfg)
    else:
        attended, amask = G._encoder(icfg, p, _bottom_torch(cfg, p, x), m)
    if cfg.get("attention_type") == "content":
        costs = CO._cost_matrix_torch(icfg, p, attended, amask, labels, lm)
    else:
        costs = G._cost_matrix(icfg, p, attended, amask, labels, lm)
    cost = costs.sum() / labels.shape[1]
    if decay > 0:
        cost = cost + decay * sum((v ** 2).sum() for k, v in p.items() if G.is_weight(k))
    grads = torch.autograd.grad(cost, list(p.values()), allow_unused=True)
    out = OrderedDict((k, np.zeros(v.shape) if g is None else g.numpy().copy()) for (k, v), g in zip(p.items(), grads))
    if return_costs:
        return float(cost.detach()), out, costs.detach().numpy()
    return float(cost.detach()), out


def train_step(cfg, params, state, batch, tc):
    """G.train_step with the bottom: gradients, then the oracle's step rules."""
    cost, grads = cost_and_grads(cfg, params, *batch, decay=tc.get("decay", 0.0))
    p64 = OrderedDict((k, np.asarray(v, dtype=np.float64)) for k, v in params.items())
    steps = G.apply_step_rules(p64, grads, state, tc)
    return OrderedDict((k, p64[k] - steps[k]) for k in p64), cost, grads


def kinks(cfg, params, recordings, recordings_mask, eps=1e-5):
    """(layer, frame, row, unit) of every Rectifier pre-activation of a live frame within eps of 0 (a float32 value
    there may land on either side of the kink); [] for Tanh."""
    if cfg["bottom"]["activation"] != "relu":
        return []
    live = np.ones(recordings.shape[:2], bool) if recordings_mask is None else np.asarray(recordings_mask) > 0
    out = []
    for i, z in enumerate(pre_activations(cfg, params, np.asarray(recordings, np.float64))):
        out += [(i,) + tuple(int(v) for v in j) for j in np.argwhere((np.abs(z) < eps) & live[:, :, None])]
    return out
