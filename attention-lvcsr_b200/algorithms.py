"""Training algorithm surface of the reference over the CUDA training step.

Mirrors ``blocks.algorithms`` as lvsr uses it (lvsr/main.py:480-519): the step rules are
configuration objects with the reference's names and constructor arguments,
``GradientDescent(...).process_batch(batch)`` runs one update
(libs/blocks/blocks/algorithms/__init__.py:244-256,284-287).  No symbolic graph exists: the chain
is mapped onto ``lvsr_train_config`` and executed by ``lvsr_train_cost_and_grads`` /
``lvsr_train_apply_updates`` (include/lvsr_b200.h).  A chain the CUDA step does not implement raises
``NotImplementedError`` instead of being approximated.

Data parallelism (SURVEY.md 8e; the reference is single-device): with ``torch.distributed``
initialised, every rank computes the gradient SUM of its utterance shard, ONE all-reduce carries the
flat gradient buffer together with the local batch size and cost, and every replica applies the same
update with 1 / (global batch size).
"""
import ctypes as C
import logging
from collections import OrderedDict

import numpy as np

from . import _lib

logger = logging.getLogger(__name__)

# Adaptive weight noise (lvsr/graph.py:71-251): the log-variance of parameter p belongs to the top-level
# NoiseBrick(name='adaptive_noise') and is named after p's owner path without the leading slash (graph.py:57-68,
# 173-177), so Model.get_parameter_dict (B/model.py:78-88, B/select.py:199-220) calls it
# "/adaptive_noise.recognizer/encoder/bidir0/forward/fork/fork_inputs.W".
NOISE_BRICK = "adaptive_noise"
ADAPTIVE_NOISE_DEFAULTS = dict(init_sigma=1e-6, model_cost_coefficient=1.0, seed=None)   # graph.py:71-80
# regularization.dropout / noise / penalty_coof (lvsr/main.py:400-417); seed None or 0 is Blocks' default_seed, 1
REGULARIZATION_DEFAULTS = dict(dropout=False, noise=0.0, penalty_coof=0.0, seed=None)
GREEDY_EXTRA_STEPS = 10       # LVSR_GREEDY_EXTRA_STEPS: greedy exploration generates L + 10 steps (lvsr/main.py:251)
ADAPTIVE_NOISE_ERROR = "using  adaptive noise with alignment weight panalty or weight decay is probably stupid"


def noise_parameter_name(name):
    """Blocks name of the adaptive-noise log-variance of the parameter called `name`."""
    return "/%s.%s" % (NOISE_BRICK, name.lstrip("/"))


class StepRule(object):
    pass


class StepClipping(StepRule):
    """B/algorithms/__init__.py:610-643.

    ``adaptive`` (set by ``adaptive_clipping``): None, or dict(burnin_period, decay_rate) of the AdaptiveClipping
    extension that resets this rule's threshold after every batch (lvsr/extensions.py:64-91); ``threshold`` is then its
    initial threshold."""

    def __init__(self, threshold=None):
        self.threshold = threshold
        self.adaptive = None
        self._recognizer = None

    def current_threshold(self):
        """The threshold the next update uses: under adaptive clipping the device value once a GradientDescent has
        been initialised with this rule (lvsr_train_clipping_threshold; synchronises), else ``threshold``."""
        if self.adaptive is None or self._recognizer is None:
            return None if self.threshold is None else float(self.threshold)
        v = C.c_double()
        _lib.check(_lib.load().lvsr_train_clipping_threshold(self._recognizer._require_ready(), C.byref(v)))
        return float(v.value)


def adaptive_clipping(step_rule, burnin_period=100, decay_rate=0.99):
    """Mark the StepClipping of `step_rule` (a StepClipping, or a CompositeRule holding one) as adaptive, as
    ``AdaptiveClipping(total_gradient_norm, clipping, gradient_threshold, decay_rate, burnin_period)`` does in
    lvsr/main.py:616-619 (defaults: lvsr/extensions.py:66-67; lvsr/main.py passes 0.998 and 500).  Returns `step_rule`.
    GradientDescent.initialize() then keeps the threshold's statistics on the device (include/lvsr_b200.h)."""
    comps = step_rule.components if isinstance(step_rule, CompositeRule) else [step_rule]
    clips = [c for c in comps if isinstance(c, StepClipping)]
    if len(clips) != 1:
        raise ValueError("adaptive_clipping needs exactly one StepClipping in the rule, found %d" % len(clips))
    if not clips[0].threshold or clips[0].threshold <= 0:
        raise ValueError("adaptive_clipping needs an initial threshold > 0, got %r" % (clips[0].threshold,))
    if int(burnin_period) < 1 or not 0.0 <= float(decay_rate) <= 1.0:
        raise ValueError("adaptive_clipping: burnin_period >= 1 and decay_rate in [0, 1] expected")
    clips[0].adaptive = dict(burnin_period=int(burnin_period), decay_rate=float(decay_rate))
    return step_rule


def clipping_rule(step_rule):
    """The StepClipping of `step_rule`, or None."""
    comps = step_rule.components if isinstance(step_rule, CompositeRule) else [step_rule]
    return next((c for c in comps if isinstance(c, StepClipping)), None)


class Scale(StepRule):
    def __init__(self, learning_rate=1.0):
        self.learning_rate = learning_rate


class BasicMomentum(StepRule):
    def __init__(self, momentum=0.0):
        self.momentum = momentum


class Momentum(StepRule):
    """Scale(learning_rate) then BasicMomentum(momentum), B/algorithms/__init__.py:431-461."""

    def __init__(self, learning_rate=1.0, momentum=0.0):
        self.learning_rate = learning_rate
        self.momentum = momentum


class AdaDelta(StepRule):
    """:464-516."""

    def __init__(self, decay_rate=0.95, epsilon=1e-6):
        if not 0.0 <= decay_rate <= 1.0:
            raise ValueError("decay rate needs to be in [0, 1]")
        self.decay_rate = decay_rate
        self.epsilon = epsilon


class VariableClipping(StepRule):
    """:646-720; the CUDA step implements axis=0 (the only use in lvsr/main.py:503-505)."""

    def __init__(self, threshold, axis=None):
        self.threshold = threshold
        self.axis = axis


class Restrict(StepRule):
    """:864-893.  ``variables``: parameter names, or the string "WEIGHT" for every parameter with the
    WEIGHT role (what lvsr/main.py:492 selects)."""

    def __init__(self, step_rule, variables="WEIGHT"):
        self.step_rule = step_rule
        self.variables = variables


class RemoveNotFinite(StepRule):
    """:829-861.  lvsr passes scaler=0.0 (lvsr/main.py:516): a parameter whose step is not finite is ZEROED."""

    def __init__(self, scaler=1):
        self.scaler = scaler


class BurnIn(StepRule):
    """lvsr/algorithms.py:19-43."""

    def __init__(self, num_steps=0):
        self.num_steps = num_steps


class CompositeRule(StepRule):
    def __init__(self, components):
        self.components = list(components)


def step_rule_from_config(train_conf, reg_conf=None):
    """The CompositeRule lvsr/main.py:480-516 builds from config['training'] / config['regularization']."""
    reg_conf = reg_conf or {}
    rules = [StepClipping(train_conf["gradient_threshold"])]
    names = train_conf.get("rules", ["momentum"])
    if "momentum" in names:
        rules.append(Momentum(train_conf["scale"], train_conf["momentum"]))
    if "adadelta" in names:
        rules.append(AdaDelta(train_conf["decay_rate"], train_conf["epsilon"]))
    if reg_conf.get("max_norm", False) > 0:
        if reg_conf.get("max_norm_exclude_lookup", False):
            raise NotImplementedError("max_norm_exclude_lookup (lvsr/main.py:494-496): the CUDA step clips every "
                                      "WEIGHT parameter, the lookup table included")
        rules.append(Restrict(VariableClipping(reg_conf["max_norm"], axis=0), "WEIGHT"))
    rules.append(RemoveNotFinite(0.0))
    if train_conf.get("burn_in_steps", 0):
        rules.append(BurnIn(num_steps=train_conf["burn_in_steps"]))
    return CompositeRule(rules)


LvsrTrainConfig = _lib.LvsrTrainConfig


def _to_train_config(step_rule, decay=0.0):
    """Accepts exactly the chain shapes lvsr/main.py can build, in that order."""
    comps = step_rule.components if isinstance(step_rule, CompositeRule) else [step_rule]
    cfg = LvsrTrainConfig()
    cfg.gradient_threshold = 0.0
    cfg.decay = float(decay)
    stage = 0          # 0 clipping, 1 momentum, 2 adadelta, 3 max-norm, 4 remove-not-finite, 5 burn-in
    seen_rnf = False
    for r in comps:
        if isinstance(r, StepClipping) and stage <= 0:
            cfg.gradient_threshold = float(r.threshold or 0.0)
            stage = 1
        elif isinstance(r, Momentum) and stage <= 1:
            cfg.use_momentum, cfg.scale, cfg.momentum = 1, float(r.learning_rate), float(r.momentum)
            stage = 2
        elif isinstance(r, Scale) and stage <= 1:
            cfg.use_momentum, cfg.scale, cfg.momentum = 1, float(r.learning_rate), 0.0
            stage = 2
        elif isinstance(r, AdaDelta) and stage <= 2:
            cfg.use_adadelta, cfg.decay_rate, cfg.epsilon = 1, float(r.decay_rate), float(r.epsilon)
            stage = 3
        elif isinstance(r, Restrict) and stage <= 3 and isinstance(r.step_rule, VariableClipping) and \
                r.variables == "WEIGHT" and r.step_rule.axis == 0:
            cfg.max_norm = float(r.step_rule.threshold)
            stage = 4
        elif isinstance(r, RemoveNotFinite) and stage <= 4:
            if r.scaler != 0.0:
                raise NotImplementedError("RemoveNotFinite(scaler=%r): the CUDA step implements scaler=0.0 "
                                          "(lvsr/main.py:516)" % (r.scaler,))
            seen_rnf = True
            stage = 5
        elif isinstance(r, BurnIn) and stage <= 5:
            cfg.burn_in_steps = int(r.num_steps)
            stage = 6
        else:
            raise NotImplementedError("step rule chain %s is not one lvsr/main.py:480-516 builds"
                                      % [type(c).__name__ for c in comps])
    if not seen_rnf:
        raise NotImplementedError("the CUDA step always applies RemoveNotFinite(0.0) (lvsr/main.py:516): add it to the chain")
    return cfg


def allreduce_step_buffer(buf, n, local_batch, local_cost, dist):
    """The ONE collective of a data-parallel training step (SURVEY.md 8e): sum over ranks of
    [flat gradient (n floats) | local batch size | local cost sum].  ``buf`` is a 1-D float32 tensor of at
    least n + 2 elements on any device ``dist`` can reduce (NCCL: the GPU buffer the backward pass wrote;
    gloo: a CPU tensor in the host-side tests).  Returns (global batch size, global cost sum) as 0-d tensors
    that live in ``buf`` -- reading them on the host synchronises."""
    buf[n] = float(local_batch)
    buf[n + 1:n + 2] = local_cost.reshape(1).to(buf.dtype) if hasattr(local_cost, "reshape") else float(local_cost)
    dist.all_reduce(buf, op=dist.ReduceOp.SUM)
    return buf[n], buf[n + 1]


def _regularization(reg):
    """The checked `regularization` argument of GradientDescent -> dict(dropout, noise, penalty_coof, seed), or None
    when none of the three is on.  Like lvsr/main.py:402-408, which builds the noisy graph from the clean one, weight
    noise discards dropout: dropout is then logged and dropped."""
    unknown = set(reg) - set(REGULARIZATION_DEFAULTS)
    if unknown:
        raise TypeError("regularization: unknown arguments %s" % sorted(unknown))
    r = dict(REGULARIZATION_DEFAULTS, **reg)
    if not isinstance(r["dropout"], bool):
        raise TypeError("regularization: dropout must be a bool, got %r" % (r["dropout"],))
    noise = float(r["noise"])
    if not (np.isfinite(noise) and noise >= 0.0):
        raise ValueError("regularization: noise must be a standard deviation >= 0, got %r" % (r["noise"],))
    coof = float(r["penalty_coof"])
    if not (np.isfinite(coof) and coof >= 0.0):
        raise ValueError("regularization: penalty_coof must be >= 0, got %r" % (r["penalty_coof"],))
    dropout = r["dropout"]
    if dropout and noise > 0:
        logger.warning("regularization: dropout has no effect with noise (the reference applies the noise to the graph "
                       "without dropout, lvsr/main.py:402-408): dropped")
        dropout = False
    if not (dropout or noise > 0 or coof > 0):
        return None
    return dict(dropout=dropout, noise=noise, penalty_coof=coof, seed=int(r["seed"] or 1))


def check_trainable_net(net):
    """Refuse a config['net'] the training step cannot run: a stacked decoder (dec_stack > 1) decodes and scores, but
    has no backward pass."""
    if net.get("dec_stack", 1) != 1:
        raise NotImplementedError("attention-lvcsr_b200: training with dec_stack=%d (a stacked decoder is inference "
                                  "only: cost, analyze, beam search and sampling)" % net["dec_stack"])


# config['training']['exploration'] values the training step runs (lvsr/main.py:245-283); 'mixed' also draws, per
# utterance, whether to train on the labels or on the greedy prediction
EXPLORATIONS = ("imitative", "greedy")


def check_exploration(net, exploration, regularization=None):
    """The exploration a training step of `net` (config['net'] with its criterion) runs for config['training']'s
    `exploration` (None: the reference's default, imitative), refused before any device work when the step cannot run
    it.  Only a task-loss criterion (mse_gain / mse_reward) reads the key: a log-likelihood model trains on its labels
    whatever it says.  `regularization`: the dropout / noise / penalty_coof the step applies (None: none, as under
    adaptive noise, which drops them)."""
    if (net.get("criterion") or {}).get("name", "log_likelihood") == "log_likelihood":
        return "imitative"
    exploration = exploration or "imitative"
    if exploration == "mixed":
        raise NotImplementedError("attention-lvcsr_b200: exploration 'mixed' (lvsr/main.py:262-276) is not built: "
                                  "use 'imitative' or 'greedy'")
    if exploration not in EXPLORATIONS:
        raise ValueError("unknown exploration %r (lvsr/main.py:279-280 accepts imitative, greedy and mixed)"
                         % (exploration,))
    reg = _regularization(regularization or {})
    if exploration == "greedy" and reg:
        if reg["penalty_coof"] > 0:
            raise ValueError("greedy exploration with penalty_coof > 0: the alignment penalty pairs the L + 10 "
                             "generated steps with the L-row labels mask (lvsr/main.py:411-417)")
        if reg["dropout"]:
            raise NotImplementedError("greedy exploration with dropout: the reference's dropout graph holds two "
                                      "applications of the bottom, in no defined order (lvsr/main.py:400-408)")
    return exploration


class GradientDescent(object):
    """``GradientDescent(cost=..., parameters=..., step_rule=...)`` of the reference with the recognizer in
    place of the symbolic cost (there is no graph to differentiate: the backward pass is part of the library).

    recognizer: attention_lvcsr_b200.SpeechRecognizer;  step_rule: CompositeRule as built by lvsr/main.py;
    decay: config['regularization']['decay'] (lvsr/main.py:419-421).

    ``last_cost`` after ``process_batch`` is the reference's ``sequence_total_cost``, sum(cost_matrix) / batch size
    (lvsr/main.py:340-344), WITHOUT the decay term: the gradient includes decay * ||WEIGHT parameters||^2, the reported
    cost does not (it is ``train_cost`` minus that penalty), so costs stay comparable across decay settings and
    no extra reduction over the parameters runs per step.

    adaptive_noise: config['regularization']['adaptive_noise'] plus ``num_examples`` (lvsr/main.py:425-437):
    dict(num_examples, init_sigma=1e-6, model_cost_coefficient=1.0, seed=None); seed None or 0 is Blocks'
    default_seed, 1.  Every step then runs forward and backward on parameters perturbed by Gaussian noise whose
    log-variances are trained with the parameters (lvsr/graph.py:71-251; include/lvsr_b200.h).  Decay has no effect
    on the step under adaptive noise: like the reference, an error is logged and decay is dropped.  ``last_cost``
    stays the task cost; ``last_model_cost``, ``model_prior_mean`` and ``model_prior_variance`` report the rest.
    Inference (cost, search, sampling) always uses the means.

    regularization: config['regularization']'s dropout, noise and penalty_coof, plus a seed:
    dict(dropout=False, noise=0.0, penalty_coof=0.0, seed=None) (lvsr/main.py:400-417).  ``dropout`` (a bool, the
    schema's type) multiplies the encoder's input, the recordings or the bottom MLP's output, by Bernoulli(0.5) / 0.5
    in every training step; ``noise`` > 0 adds N(0, noise^2) to every parameter outside the attention for forward and
    backward, and the gradient there updates the clean parameters.  Fresh draws every update, keyed by (seed, update,
    global utterance index) and (seed, update, parameter element); include/lvsr_b200.h.  With noise on, dropout is
    dropped with a warning, as the reference builds its noisy graph from the graph without dropout.  ``penalty_coof``
    > 0 adds penalty_coof * weights_penalty / B to the cost the gradient is taken of, weights_penalty being the
    alignment monotonicity penalty of the regularised forward (lvsr/expressions.py:14-19, lvsr/main.py:411-417).
    Under adaptive noise the reference trains on the clean graph, so all three are dropped with a logged error.
    Data-parallel dropout needs equal shards: rank r's first utterance is utterance r * B of the global batch.
    ``last_cost`` stays the task cost of the regularised forward; ``last_penalty`` is weights_penalty / B of the
    last update (a device scalar; None when the penalty is off), all-reduced with the gradient.

    exploration: config['training']['exploration'] (check_exploration), read under a task-loss criterion only.
    'imitative' trains on the labels; 'greedy' generates L + 10 steps of the model's own arg-max output on the device
    with the parameters the step runs on, and trains on that prediction scored against the labels (lvsr/main.py:
    245-283).  ``last_prediction`` is then (prediction [L + 10, B] int64, its mask [L + 10, B] float32), device tensors
    of the last step; None otherwise.  Each data-parallel rank explores its own shard."""

    def __init__(self, recognizer=None, step_rule=None, decay=0.0, cost=None, parameters=None, gradients=None,
                 on_unused_sources="warn", adaptive_noise=None, regularization=None, exploration="imitative",
                 **kwargs):
        if recognizer is None:
            raise ValueError("GradientDescent needs the recognizer (no symbolic cost exists in the CUDA path)")
        if getattr(recognizer, "lm", None):
            # with an LM the reference's emitter is LMEmitter, whose costs are the fused readout's: inference only
            raise NotImplementedError("attention-lvcsr_b200: training with a language model (shallow fusion is "
                                      "inference only)")
        net = dict(getattr(recognizer, "net", {}), criterion=getattr(recognizer, "criterion", None))
        check_trainable_net(net)
        self.exploration = check_exploration(net, exploration, None if adaptive_noise else regularization)
        self.recognizer = recognizer
        self.step_rule = step_rule if step_rule is not None else CompositeRule([Scale(), RemoveNotFinite(0.0)])
        self.adaptive_noise = None
        if adaptive_noise:
            unknown = set(adaptive_noise) - set(ADAPTIVE_NOISE_DEFAULTS) - {"num_examples"}
            if unknown:
                raise TypeError("adaptive_noise: unknown arguments %s" % sorted(unknown))
            if "num_examples" not in adaptive_noise:
                raise ValueError("adaptive_noise needs num_examples, the size of the training set (lvsr/main.py:434)")
            an = dict(ADAPTIVE_NOISE_DEFAULTS, **adaptive_noise)
            self.adaptive_noise = dict(num_examples=int(an["num_examples"]), init_sigma=float(an["init_sigma"]),
                                       model_cost_coefficient=float(an["model_cost_coefficient"]),
                                       seed=int(an["seed"] or 1))
        self.regularization = _regularization(regularization or {})
        if self.adaptive_noise:
            # lvsr/main.py:425-437: the cost and its gradients are rebuilt from the clean graph, so decay and the three
            # regularisers have no effect; the reference logs the error below for the penalty and decay
            coof = float((regularization or {}).get("penalty_coof", 0.0))
            if decay > 0 or coof > 0:
                logger.error(ADAPTIVE_NOISE_ERROR)
            if self.regularization:
                logger.error("regularization %s has no effect under adaptive noise: dropped", self.regularization)
            decay = 0.0
            self.regularization = None
        self._tc = _to_train_config(self.step_rule, decay)
        self.on_unused_sources = on_unused_sources
        self._grads = None
        self._buf = None
        self._cost = None
        self.equal_shards = True
        self.last_cost = None
        self.last_penalty = None
        self.last_batch_size = None
        self.last_prediction = None

    SOURCES = ("recordings", "recordings_mask", "labels", "labels_mask")

    def initialize(self):
        rec = self.recognizer
        torch = rec._torch()
        lib, h = _lib.load(), rec._require_ready()
        n = int(lib.lvsr_model_flat_size(h))
        # [flat gradient | local batch size | local cost sum | penalty sum | padding]: one buffer, one all-reduce
        self._buf = torch.zeros((n + 64,), dtype=torch.float32, device=rec.device)
        self._cost = torch.zeros((1,), dtype=torch.float32, device=rec.device)
        self._n = n
        _lib.check(lib.lvsr_train_reset(h))
        clip = clipping_rule(self.step_rule)
        if clip is not None and getattr(clip, "adaptive", None) is not None:
            cfg = _lib.LvsrAdaptiveClipping(initial_threshold=float(clip.threshold),
                                            decay_rate=clip.adaptive["decay_rate"],
                                            burnin_period=clip.adaptive["burnin_period"])
            _lib.check(lib.lvsr_train_set_adaptive_clipping(h, C.byref(cfg)))
            clip._recognizer = rec
        else:
            _lib.check(lib.lvsr_train_set_adaptive_clipping(h, None))
        if self.adaptive_noise:
            an = self.adaptive_noise
            cfg = _lib.LvsrAdaptiveNoise(init_sigma=an["init_sigma"], model_cost_coefficient=an["model_cost_coefficient"],
                                         num_examples=an["num_examples"], seed=an["seed"])
            _lib.check(lib.lvsr_train_set_adaptive_noise(h, C.byref(cfg)))
            self._noise_grads = torch.zeros((n,), dtype=torch.float32, device=rec.device)
        if self.regularization:
            r = self.regularization
            cfg = _lib.LvsrRegularization(dropout=int(r["dropout"]), noise_level=r["noise"],
                                          penalty_coof=r["penalty_coof"], seed=r["seed"])
            _lib.check(lib.lvsr_train_set_regularization(h, C.byref(cfg)))
        else:
            _lib.check(lib.lvsr_train_set_regularization(h, None))

    def _world(self):
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            return dist, dist.get_world_size()
        return None, 1

    def cost_and_gradients(self, batch):
        """(cost, {parameter name: gradient}) of sum(cost_matrix)/B for this batch on this GPU (no update).  Under
        adaptive noise: the gradients of the reference (lvsr/graph.py:238-249) at this update's noise, the means'
        first, then the log-variances' under their Blocks names."""
        rec = self.recognizer
        if self._buf is None:
            self.initialize()
        B = self._forward_backward(batch, None)
        import ctypes as C_
        lib, h = _lib.load(), rec._require_ready()
        if self.adaptive_noise:
            _lib.check(lib.lvsr_train_noise_gradients(h, self._buf.data_ptr(), 1.0, self._noise_grads.data_ptr(),
                                                      rec._stream()))
        flat = self._buf[:self._n].cpu().numpy()
        out = OrderedDict()
        for (name, (off, cnt)), shape in zip(self._offsets().items(), rec.parameter_shapes().values()):
            out[name] = flat[off:off + cnt].reshape(shape).copy()
        if self.adaptive_noise:
            flat = self._noise_grads.cpu().numpy()
            for (name, (off, cnt)), shape in zip(self._offsets().items(), rec.parameter_shapes().values()):
                out[noise_parameter_name(name)] = flat[off:off + cnt].reshape(shape).copy()
        return float(self._cost.item()), out

    def _offsets(self):
        """{parameter name: (flat offset, element count)}."""
        lib, h = _lib.load(), self.recognizer._require_ready()
        out = OrderedDict()
        for i in range(lib.lvsr_model_num_params(h)):
            off, cnt = C.c_int64(), C.c_int64()
            _lib.check(lib.lvsr_model_param_offset(h, i, C.byref(off), C.byref(cnt)))
            out[lib.lvsr_model_param_name(h, i).decode()] = (off.value, cnt.value)
        return out

    # ---- adaptive weight noise ------------------------------------------------------------------------------------
    def _require_noise(self):
        if not self.adaptive_noise:
            raise RuntimeError("adaptive noise is off (GradientDescent(adaptive_noise=...))")
        if self._buf is None:
            self.initialize()
        return _lib.load(), self.recognizer._require_ready()

    def noise_parameter_values(self):
        """{Blocks name of the noise parameter ("/adaptive_noise.recognizer/..."): log-variance ndarray}."""
        lib, h = self._require_noise()
        out = OrderedDict()
        for i, (name, shape) in enumerate(self.recognizer.parameter_shapes().items()):
            arr = np.empty(shape, dtype=np.float32)
            _lib.check(lib.lvsr_train_get_noise_param(h, i, arr.ctypes.data, arr.size))
            out[noise_parameter_name(name)] = arr
        return out

    def set_noise_parameter_values(self, values):
        """Set log-variances by their Blocks names; the others keep their values."""
        lib, h = self._require_noise()
        index = OrderedDict((noise_parameter_name(n), (i, s))
                            for i, (n, s) in enumerate(self.recognizer.parameter_shapes().items()))
        for name, value in values.items():
            if name not in index:
                raise KeyError("unknown noise parameter %s" % name)
            i, shape = index[name]
            arr = np.ascontiguousarray(value, dtype=np.float32)
            if tuple(arr.shape) != shape:
                raise ValueError("noise parameter %s: expected shape %s, got %s" % (name, shape, arr.shape))
            _lib.check(lib.lvsr_train_set_noise_param(h, i, arr.ctypes.data, arr.size))

    def noise_stats(self):
        """{model_cost, model_prior_mean, model_prior_variance} of the last training forward (synchronises)."""
        lib, h = self._require_noise()
        out = (C.c_double * 3)()
        _lib.check(lib.lvsr_train_noise_stats(h, out))
        return OrderedDict(zip(_lib.NOISE_STATS, (float(v) for v in out)))

    @property
    def last_model_cost(self):
        return self.noise_stats()["model_cost"] if self.adaptive_noise else None

    @property
    def model_prior_mean(self):
        return self.noise_stats()["model_prior_mean"] if self.adaptive_noise else None

    @property
    def model_prior_variance(self):
        return self.noise_stats()["model_prior_variance"] if self.adaptive_noise else None

    def _forward_backward(self, batch, gscale, utterance_offset=0):
        rec = self.recognizer
        torch = rec._torch()
        lib, h = _lib.load(), rec._require_ready()
        batch = dict(batch)
        unknown = set(batch) - set(self.SOURCES)
        if unknown and self.on_unused_sources == "raise":
            raise ValueError("mismatch of variable names and data sources: %s" % sorted(unknown))
        missing = [s for s in ("recordings", "labels") if s not in batch]
        if missing:
            raise ValueError("Didn't find all sources: %s" % missing)
        x = rec._dev(batch["recordings"], torch.float32)
        m = rec._dev(batch.get("recordings_mask"), torch.float32)
        rec._check_labels(batch["labels"])
        y = rec._dev(batch["labels"], torch.int64)
        ym = rec._dev(batch.get("labels_mask"), torch.float32)
        if x.dim() != 3 or y.dim() != 2:
            raise ValueError("recordings [T,B,F] and labels [L,B] expected")
        T, B, F = x.shape
        L = y.shape[0]
        if F != rec.net["num_features"] or y.shape[1] != B or (m is not None and tuple(m.shape) != (T, B)) or \
                (ym is not None and tuple(ym.shape) != (L, B)):
            raise ValueError("batch shapes disagree: recordings %s mask %s labels %s labels_mask %s" % (
                tuple(x.shape), None if m is None else tuple(m.shape), tuple(y.shape), None if ym is None else tuple(ym.shape)))
        gs = (1.0 / B) if gscale is None else gscale
        if self.regularization and self.regularization["dropout"]:
            _lib.check(lib.lvsr_train_set_utterance_offset(h, int(utterance_offset)))
        if self.exploration == "greedy":
            n = L + GREEDY_EXTRA_STEPS
            pred = torch.empty((n, B), dtype=torch.int64, device=rec.device)
            pmask = torch.empty((n, B), dtype=torch.float32, device=rec.device)
            _lib.check(lib.lvsr_train_cost_and_grads_greedy(
                h, x.data_ptr(), None if m is None else m.data_ptr(), y.data_ptr(), T, B, L, float(gs),
                self._cost.data_ptr(), self._buf.data_ptr(), pred.data_ptr(), pmask.data_ptr(), rec._stream()))
            self.last_prediction = (pred, pmask)
        else:
            _lib.check(lib.lvsr_train_cost_and_grads(
                h, x.data_ptr(), None if m is None else m.data_ptr(), y.data_ptr(), None if ym is None else ym.data_ptr(),
                T, B, L, float(gs), self._cost.data_ptr(), self._buf.data_ptr(), rec._stream()))
        if self._penalty_on():
            # the penalty sum rides in the step buffer's padding: the data-parallel step stays one all-reduce
            _lib.check(lib.lvsr_train_penalty_sum(h, self._buf.data_ptr() + 4 * (self._n + 2), rec._stream()))
        return B

    def process_batch(self, batch):
        """One update (B/algorithms/__init__.py:284-287): parameters change in place on the device."""
        rec = self.recognizer
        if self._buf is None:
            self.initialize()
        lib, h = _lib.load(), rec._require_ready()
        dist, world = self._world()
        if world == 1:
            B = self._forward_backward(batch, None)          # grads already carry 1/B
            _lib.check(lib.lvsr_train_apply_updates(h, self._buf.data_ptr(), 1.0, C.byref(self._tc), rec._stream()))
            self.last_batch_size = B
            self.last_cost = self._cost                       # device scalar; .item() synchronises
            self.last_penalty = self._buf[self._n + 2] / B if self._penalty_on() else None
            return
        B = self._forward_backward(batch, 1.0, self._utterance_offset(dist, batch))   # gradient SUM over the local utterances
        bg_dev, cost_dev = allreduce_step_buffer(self._buf, self._n, B, self._cost, dist)   # the ONE collective of the step
        # the global batch size has to reach the host to become a kernel argument; every rank knows its own B and
        # shards are equal-sized in the data-parallel loop, so the common case needs no synchronisation
        Bg = B * world if self.equal_shards else int(round(float(bg_dev.item())))
        _lib.check(lib.lvsr_train_apply_updates(h, self._buf.data_ptr(), 1.0 / Bg, C.byref(self._tc), rec._stream()))
        self.last_batch_size = Bg
        self.last_cost = cost_dev / Bg
        self.last_penalty = self._buf[self._n + 2] / Bg if self._penalty_on() else None

    def _penalty_on(self):
        return bool(self.regularization and self.regularization["penalty_coof"] > 0)

    def _utterance_offset(self, dist, batch):
        """Global index of this rank's first utterance, the key of its dropout mask: rank * B under equal shards."""
        if not (self.regularization and self.regularization["dropout"]):
            return 0
        if not self.equal_shards:
            # with unequal shards the offset takes a second collective (a scan of the shard sizes) besides the step's
            # one all-reduce
            raise NotImplementedError("data-parallel dropout keys its mask by global utterance index, which needs "
                                      "equal shards (equal_shards=True): rank r's first utterance is r * B")
        return dist.get_rank() * len(batch["recordings"][0])

    def total_gradient_norm(self):
        lib, h = _lib.load(), self.recognizer._require_ready()
        v = C.c_float()
        _lib.check(lib.lvsr_train_gradient_norm(h, C.byref(v)))
        return float(v.value)
