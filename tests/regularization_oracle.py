"""Float64 oracle of dropout and weight noise (regularization.dropout / noise) -- TEST INFRASTRUCTURE ONLY.

lvsr/main.py:400-408 regularises the training graph with Blocks' apply_dropout and apply_noise:
  * dropout: the bottom's output (the recordings without a bottom MLP) becomes x * mask / (1 - p), mask ~
    Bernoulli(1 - p), p = 0.5, over every element (B/graph/__init__.py:425-540);
  * noise: every parameter outside Selector(generator.transition.attention) becomes p + N(0, level^2)
    (B/graph/__init__.py:312-336; lvsr/main.py:297-298,405-408).
  * penalty_coof: train_cost += coof * weights_penalty / B (lvsr/main.py:411-417), weights_penalty the monotonicity
    penalty of the regularised forward's alignments (lvsr/expressions.py:14-19), whose max(., 0) has Theano's
    gradient eq(output, x): a tie counts as 1.
The draws are the library's own (replayed through lvsr_train_dropout_mask / lvsr_train_weight_noise_sample), so the
oracle takes the multiplier and eps as inputs.  Gradients are taken at the regularised point and belong to the clean
parameters (p + level eps is p plus a constant).
"""
from collections import OrderedDict

import numpy as np

from oracle import lvsr_oracle_grad as G
import bottom_oracle as BO
import content_oracle as CO

ATTENTION = ("/recognizer/generator/att_trans/conv_att/", "/recognizer/generator/att_trans/cont_att/")
DROPOUT_P = 0.5


def is_noise_subject(name):
    """Blocks' apply_noise subjects of lvsr/main.py: every parameter that is not the attention's."""
    return not name.startswith(ATTENTION)


def dropout(x, mask, p=DROPOUT_P):
    """apply_dropout's replacement of x: x * mask / (1 - p)."""
    return np.asarray(x, np.float64) * np.asarray(mask, np.float64) / (1.0 - p)


def noisy(params, eps, level):
    """apply_noise's replacement of every subject p: p + level eps; the attention's parameters as they are."""
    return OrderedDict((k, np.asarray(v, np.float64) + (level * np.asarray(eps[k], np.float64) if is_noise_subject(k)
                                                         else 0.0)) for k, v in params.items())


def penalty(w, labels_mask=None):
    """weights_penalty = sum_b sum_{i>=1} m[i,b] sum_t max(c_i[t] - c_{i-1}[t], 0), c_i = cumsum_t w_i, of alignments
    w [L, B, T] (numpy or a torch tensor; with torch, the gradient of max(x, 0) is [x >= 0])."""
    if isinstance(w, np.ndarray):
        c = np.cumsum(np.asarray(w, np.float64), axis=2)
        d = np.maximum(c[1:] - c[:-1], 0.0).sum(axis=2)
        m = np.ones(d.shape) if labels_mask is None else np.asarray(labels_mask, np.float64)[1:]
        return float((d * m).sum())
    import torch
    c = torch.cumsum(w, dim=2)
    diff = c[1:] - c[:-1]
    d = (diff * (diff >= 0).to(diff.dtype)).sum(dim=2)
    return d.sum() if labels_mask is None else (d * labels_mask[1:]).sum()


def penalty_grad(w, labels_mask=None):
    """The hand-written gradient of penalty(w): dP/dw_i[t'] = sum_{t>=t'} (m_i [c_i[t] >= c_{i-1}[t]] -
    m_{i+1} [c_{i+1}[t] >= c_i[t]]), the first term absent for i = 0 and the second for i = L - 1."""
    w = np.asarray(w, np.float64)
    L = w.shape[0]
    m = np.ones(w.shape[:2]) if labels_mask is None else np.asarray(labels_mask, np.float64)
    c = np.cumsum(w, axis=2)
    up = (c[1:] >= c[:-1]).astype(np.float64) * m[1:, :, None]      # [c_i >= c_{i-1}] m_i, i >= 1
    g = np.zeros_like(w)
    g[1:] += up
    g[:L - 1] -= up
    return np.cumsum(g[:, :, ::-1], axis=2)[:, :, ::-1]


class _Alignments(object):
    """Records the alignments [B, T] of every step while the torch mirror runs its cost matrix."""

    def __init__(self, content):
        self.content, self.rows = content, []

    def __enter__(self):
        if self.content:
            self.orig = G._compute_weights

            def wrapped(e, mask, normalizer):
                w = self.orig(e, mask, normalizer)
                self.rows.append(w.T)
                return w
            G._compute_weights = wrapped
        else:
            self.orig = G._take_glimpses

            def wrapped(*args):
                out = self.orig(*args)
                self.rows.append(out[1])
                return out
            G._take_glimpses = wrapped
        return self

    def __exit__(self, *exc):
        if self.content:
            G._compute_weights = self.orig
        else:
            G._take_glimpses = self.orig


def cost_and_grads(cfg, params, recordings, recordings_mask, labels, labels_mask, mult=None, eps=None, level=0.0,
                   coof=0.0, return_penalty=False):
    """The regularised train_cost sum(costs) / B (+ coof * weights_penalty / B) and its float64 gradient: `mult` (the
    multiplier mask / (1 - p) of the encoder's input, [T, B, F], None: no dropout), `eps` ({name: array}, None: no
    weight noise) and the penalty coefficient `coof`.  The cost returned is the task cost alone, as the library's;
    return_penalty: also weights_penalty and the alignments [L, B, T']."""
    import torch
    at = noisy(params, eps, level) if eps is not None else params
    p = OrderedDict((k, torch.tensor(np.asarray(v, dtype=np.float64), requires_grad=True)) for k, v in at.items())
    x = torch.as_tensor(np.asarray(recordings, dtype=np.float64))
    m = None if recordings_mask is None else torch.as_tensor(np.asarray(recordings_mask, dtype=np.float64))
    lm = None if labels_mask is None else torch.as_tensor(np.asarray(labels_mask, dtype=np.float64))
    labels = np.asarray(labels, dtype=np.int64)
    icfg = BO.inner(cfg)
    h = BO._bottom_torch(cfg, p, x)
    if mult is not None:
        h = h * torch.as_tensor(np.asarray(mult, dtype=np.float64))
    attended, amask = G._encoder(icfg, p, h, m)
    content = cfg.get("attention_type") == "content"
    with _Alignments(content) as al:
        if content:
            costs = CO._cost_matrix_torch(icfg, p, attended, amask, labels, lm)
        else:
            costs = G._cost_matrix(icfg, p, attended, amask, labels, lm)
    cost = costs.sum() / labels.shape[1]
    w = torch.stack(al.rows)
    pen = penalty(w, lm)
    total = cost + coof * pen / labels.shape[1] if coof > 0 else cost
    grads = torch.autograd.grad(total, list(p.values()), allow_unused=True)
    out = OrderedDict((k, np.zeros(v.shape) if g is None else g.numpy().copy()) for (k, v), g in zip(p.items(), grads))
    if return_penalty:
        return float(cost.detach()), out, float(pen.detach()), w.detach().numpy()
    return float(cost.detach()), out


def train_step(cfg, params, state, batch, tc, mult=None, eps=None, level=0.0, coof=0.0):
    """One regularised update: gradients at the regularised point, the step rules on the clean parameters."""
    cost, grads = cost_and_grads(cfg, params, *batch, mult=mult, eps=eps, level=level, coof=coof)
    p64 = OrderedDict((k, np.asarray(v, dtype=np.float64)) for k, v in params.items())
    steps = G.apply_step_rules(p64, grads, state, tc)
    return OrderedDict((k, p64[k] - steps[k]) for k in p64), cost, grads
