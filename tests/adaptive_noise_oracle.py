"""Float64 oracle of adaptive weight noise -- TEST INFRASTRUCTURE ONLY.

Restates apply_adaptive_noise (lvsr/graph.py:71-251) as lvsr/main.py:425-460,510-519 uses it, on top of the gradient
oracle (oracle/lvsr_oracle_grad.py, or tests/content_oracle.py for content attention).  For every parameter p
(graph.py:170-183), with S = 2048 (log_sigma_scale, :159):

    ls2 initialised to log(init_sigma) * 2 / S (float32),  s2 = exp(S ls2)
    p_noisy  = p + eps sqrt(s2)                                   eps is GIVEN here (the GPU's draw, replayed)
    prior_u  = sum(p) / n,  prior_s2 = (sum(s2) + sum((p - prior_u)^2)) / n        over all parameters, :186-198
    LC       = coef / N sum[0.5 (log prior_s2 - S ls2) + ((p - prior_u)^2 + s2 - prior_s2) / (2 prior_s2)]  :206-214
    g        = gradient of sum(costs) / B at p_noisy (the cost WITHOUT decay: cg.outputs[0], main.py:431-432)
    grad p   = coef (p - prior_u) / (N prior_s2) + g                                          :240-241
    grad ls2 = coef 0.5 S / N (s2 / prior_s2 - 1) + 0.5 S s2 g^2                              :243-247

The priors are constants of the gradients and g^2 stands in for the diagonal Hessian, as in the reference.  Then the
step rules of main.py:510-519 run over the union of the two groups: one StepClipping norm, Momentum / AdaDelta state
for both, RemoveNotFinite per tensor, BurnIn on both, and max-norm on the WEIGHT means only.  The oracle's
G.is_weight looks at the leaf after the last '.', so a noise name ending in '.W' would pass for a WEIGHT parameter:
the noise parameters are excluded from max-norm explicitly.

No reference test pins this code: it is unpinned by reference tests and pinned by this restatement,
tests/test_adaptive_noise_cpu.py's hand-worked known answer and its autograd check of the ls2 gradient.
"""
from collections import OrderedDict

import numpy as np

from oracle import lvsr_oracle_grad as G

LOG_SIGMA_SCALE = 2048.0
NOISE_BRICK = "adaptive_noise"


def noise_name(name):
    """Blocks name of the noise parameter of `name` (graph.py:57-68,173-177; B/select.py:199-220)."""
    return "/%s.%s" % (NOISE_BRICK, name.lstrip("/"))


def init_ls2(params, init_sigma):
    """graph.py:173-175: the float32 constant log(init_sigma) * 2 / S in every entry."""
    v = np.float32(np.log(init_sigma) * 2.0 / LOG_SIGMA_SCALE)
    return OrderedDict((k, np.full(np.shape(p), v, dtype=np.float32)) for k, p in params.items())


def priors(params, ls2):
    """(prior_u, prior_s2, LC without the coef / N factor) from the means and log-variances, float64."""
    p = {k: np.asarray(v, np.float64) for k, v in params.items()}
    s2 = {k: np.exp(LOG_SIGMA_SCALE * np.asarray(ls2[k], np.float64)) for k in p}
    n = float(sum(v.size for v in p.values()))
    u = sum(float(v.sum()) for v in p.values()) / n
    ps2 = (sum(float(s2[k].sum()) for k in p) + sum(float(((v - u) ** 2).sum()) for v in p.values())) / n
    lc = 0.0
    for k, v in p.items():
        lc += 0.5 * float((np.log(ps2) - LOG_SIGMA_SCALE * np.asarray(ls2[k], np.float64)).sum())
        lc += float(((v - u) ** 2 + s2[k] - ps2).sum()) / (2.0 * ps2)
    return u, ps2, lc


def model_cost(params, ls2, num_examples, coef):
    """(LC, prior_u, prior_s2)."""
    u, ps2, lc = priors(params, ls2)
    return lc / num_examples * coef, u, ps2


def noisy(params, ls2, eps):
    """p + eps sqrt(exp(S ls2)), float64."""
    return OrderedDict((k, np.asarray(v, np.float64) + np.asarray(eps[k], np.float64) *
                        np.sqrt(np.exp(LOG_SIGMA_SCALE * np.asarray(ls2[k], np.float64)))) for k, v in params.items())


def transform(params, ls2, grads, num_examples, coef):
    """Both gradient groups from the task gradients `grads` (at the noisy parameters): ({p: grad}, {p: grad ls2})."""
    _, u, ps2 = model_cost(params, ls2, num_examples, coef)
    gp, gl = OrderedDict(), OrderedDict()
    for k, v in params.items():
        g = np.asarray(grads[k], np.float64)
        s2 = np.exp(LOG_SIGMA_SCALE * np.asarray(ls2[k], np.float64))
        gp[k] = coef * (np.asarray(v, np.float64) - u) / (num_examples * ps2) + g
        gl[k] = coef * 0.5 / num_examples * LOG_SIGMA_SCALE * (s2 / ps2 - 1.0) + 0.5 * LOG_SIGMA_SCALE * s2 * g ** 2
    return gp, gl


def cost_and_grads(cfg, params, ls2, eps, batch, num_examples, coef):
    """Task cost and both gradient groups at p + eps sigma -> (cost, grad p, grad ls2, (LC, prior_u, prior_s2))."""
    if cfg.get("attention_type") == "content":
        import content_oracle as CO
        grad_fn = CO.cost_and_grads
    else:
        grad_fn = G.cost_and_grads
    cost, g = grad_fn(cfg, noisy(params, ls2, eps), *batch)
    gp, gl = transform(params, ls2, g, num_examples, coef)
    return cost, gp, gl, model_cost(params, ls2, num_examples, coef)


def apply_step_rules(params, ls2, gp, gl, state, tc):
    """main.py:510-519 over {p} u {ls2} -> (steps of p, steps of ls2); `state` is updated in place."""
    union = OrderedDict((k, np.asarray(v, np.float64)) for k, v in gp.items())
    union.update((noise_name(k), np.asarray(v, np.float64)) for k, v in gl.items())
    values = OrderedDict((k, np.asarray(v, np.float64)) for k, v in params.items())
    values.update((noise_name(k), np.asarray(v, np.float64)) for k, v in ls2.items())
    steps = G.step_clipping(union, tc["gradient_threshold"])
    if "momentum" in tc["rules"]:
        steps = G.momentum(steps, state, tc["scale"], tc["momentum"])
    if "adadelta" in tc["rules"]:
        steps = G.adadelta(steps, state, tc["decay_rate"], tc["epsilon"])
    if tc.get("max_norm", 0) > 0:
        steps = OrderedDict((k, G.variable_clipping(values[k], s, tc["max_norm"], axis=0)
                             if (k in params and G.is_weight(k) and s.ndim >= 1) else s) for k, s in steps.items())
    steps = OrderedDict((k, G.remove_not_finite(values[k], s, 0.0)) for k, s in steps.items())
    if tc.get("burn_in_steps", 0):
        remaining = state.setdefault("burn_in", tc["burn_in_steps"])
        mult = 1.0 if remaining <= 0 else 0.0
        steps = OrderedDict((k, s * mult) for k, s in steps.items())
        state["burn_in"] = max(0, remaining - 1)
    return (OrderedDict((k, steps[k]) for k in params), OrderedDict((k, steps[noise_name(k)]) for k in params))


def train_step(cfg, params, ls2, state, batch, tc, eps, num_examples, coef):
    """One update -> (new means, new ls2, task cost, (LC, prior_u, prior_s2), union gradient norm)."""
    cost, gp, gl, stats = cost_and_grads(cfg, params, ls2, eps, batch, num_examples, coef)
    norm = G.l2_norm(list(gp.values()) + list(gl.values()))
    sp, sl = apply_step_rules(params, ls2, gp, gl, state, tc)
    newp = OrderedDict((k, np.asarray(v, np.float64) - sp[k]) for k, v in params.items())
    newl = OrderedDict((k, np.asarray(v, np.float64) - sl[k]) for k, v in ls2.items())
    return newp, newl, cost, stats, norm
