"""SpeechRecognizer -- the reference's model object surface over the CUDA library.

Mirrors lvsr.bricks.recognizer.SpeechRecognizer (lvsr/bricks/recognizer.py:159-562):
same constructor keywords (``SpeechRecognizer(input_dims=..., input_num_chars=...,
eos_label=..., num_phonemes=..., name=..., data_prepend_eos=..., character_map=...,
**config['net'])``, lvsr/main.py:213-221), same method names and return conventions:

    initialize()                         parameters from the init schemes (reference: Blocks push/initialize)
    load_params(path) / save_params      Blocks checkpoint parameter naming (SURVEY.md 8b b4)
    cost(recordings, recordings_mask, labels, labels_mask)   -> costs [L, B]   (recognizer.py:375-390)
    analyze(inputs, groundtruth, prediction=None)            -> [costs[L], weights[L,T'], energies[L,T']]
    init_beam_search(beam_size); beam_search(inputs, **kw)   -> (outputs, costs)   (:496-533)

No symbolic graph exists: every method is a direct call into liblvsr_b200.so (C ABI in
include/lvsr_b200.h) on torch-owned device buffers.  There is no CPU fallback.
"""
import io
import logging
import tarfile
from collections import OrderedDict

import numpy as np

from . import _lib
from . import bricks as _bricks
from . import lm as _lm
from .search import BeamSearch, CandidateNotFoundError  # noqa: F401


logger = logging.getLogger(__name__)


class _Variable(object):
    """Stand-in for the Theano input variables lvsr/main.py reads the NAMES of (recognizer.inputs.keys(),
    recognizer.labels.name ...: lvsr/bricks/recognizer.py:351-361, lvsr/main.py:260-262,786)."""

    def __init__(self, name):
        self.name = name

    def __repr__(self):
        return self.name


def _ptr(t):
    return None if t is None else t.data_ptr()


# config['net']['lm'] keys and their defaults (lvsr/bricks/recognizer.py:324-331, LanguageModel's no_transition_cost)
LM_DEFAULTS = OrderedDict(weight=0.0, normalize_am_weights=True, normalize_lm_weights=False,
                          normalize_tot_weights=False, am_beta=1.0, no_transition_cost=1e12, type_="fst")


def _lm_config(lm):
    unknown = sorted(set(lm) - set(LM_DEFAULTS) - {"path"})
    if unknown:
        raise TypeError("unknown lm option(s) %s" % unknown)
    out = OrderedDict(LM_DEFAULTS)
    out.update(lm)
    if out["type_"] != "fst":
        raise ValueError("lm type_ %r: only 'fst' exists" % (out["type_"],))
    if not (out["normalize_am_weights"] or out["normalize_lm_weights"] or out["normalize_tot_weights"]):
        logger.warning("Beam search is prone to fail with no log-prob normalization")
    return out


class _Child(object):
    """Named handle into the brick tree (``recognizer.generator.transition.attention`` ...)
    for code that walks the reference's attribute paths (lvsr/main.py:297-298,354-369)."""

    def __init__(self, name, **attrs):
        self.name = name
        self.children = []
        for k, v in attrs.items():
            setattr(self, k, v)


class SpeechRecognizer(object):
    def __init__(self, input_dims, input_num_chars, eos_label, num_phonemes,
                 dim_dec, dims_bidir, enc_transition=None, dec_transition=None,
                 use_states_for_readout=True, attention_type="content_and_conv",
                 criterion=None, bottom=None, lm=None, character_map=None,
                 bidir=True, subsample=None, dims_top=None, prior=None, conv_n=None,
                 post_merge_activation=None, post_merge_dims=None, dim_matcher=None,
                 embed_outputs=True, dim_output_embedding=None, dec_stack=1,
                 conv_num_filters=1, data_prepend_eos=True, energy_normalizer=None,
                 max_decoded_length_scale=1, name="recognizer", device=None, **kwargs):
        # ---- what the CUDA path implements; everything else fails loudly ----------
        def unsupported(what):
            raise NotImplementedError("attention-lvcsr_b200: %s is outside the GPU hot path "
                                      "(SURVEY.md section 8)" % what)
        if attention_type not in _lib.ATTENTION_TYPES:
            unsupported("attention_type=%r" % attention_type)
        if lm and not lm.get("path"):
            # the reference then swaps in LMEmitter with the unfused readout: costs become raw logits
            unsupported("lm without a path")
        if lm and character_map is None:
            unsupported("lm without a character_map")
        lm = _lm_config(lm) if lm else None
        if bidir not in (True, False, 0, 1):
            # net.bidir (lvsr/configs/schema.yaml:48-49) is a boolean
            raise ValueError("bidir must be True (Bidirectional encoder layers) or False (forward-only "
                             "RecurrentWithFork layers), got %r" % (bidir,))
        if dims_top:
            unsupported("dims_top")
        if dec_stack not in (1, 2):
            # RecurrentStack of GatedRecurrent layers (lvsr/bricks/recognizer.py:250-259): one or two; two decode and
            # score only (GradientDescent refuses them)
            unsupported("dec_stack=%r (1 or 2)" % (dec_stack,))
        criterion = dict(criterion) if criterion else dict(name="log_likelihood")
        if criterion["name"] not in _lib.CRITERIA:
            raise ValueError("Unknown criterion {}".format(criterion["name"]))       # recognizer.py:297
        # with a task-loss criterion and an LM, RewardRegressionEmitter stays and reads the fused readouts
        # (lvsr/bricks/recognizer.py:285-297, 323-338): only SoftmaxEmitter is swapped for LMEmitter
        # SpeechBottom (lvsr/bricks/recognizer.py:105-157): an MLP of one Linear + activation per entry of dims, Tanh
        # when the activation is None; Identity when dims is empty
        bottom = dict(bottom or {})
        bottom.pop("bottom_class", None)
        bottom_dims = [int(d) for d in (bottom.get("dims") or [])]
        bottom_act = bottom.get("activation")
        bottom_kind = "tanh" if bottom_act is None else getattr(bottom_act, "kind", None)
        if bottom_dims and bottom_kind not in _lib.BOTTOM_ACTIVATIONS:
            unsupported("bottom MLP activation %r (Rectifier or Tanh)" % (bottom_act,))
        for tr in (enc_transition, dec_transition):
            if tr is not None and getattr(tr, "__name__", type(tr).__name__) != "GatedRecurrent":
                unsupported("transition %r" % tr)

        self.name = name
        self.eos_label = eos_label
        self.data_prepend_eos = data_prepend_eos
        self.character_map = character_map
        self.lm = lm
        self._lm_tables = _lm.load(lm["path"], character_map, int(num_phonemes)) if lm else None
        self.criterion = criterion
        self.max_decoded_length_scale = max_decoded_length_scale
        self.rec_weights_init = None
        self.initial_states_init = None
        self.weights_init = None
        self.biases_init = None
        self._brick_schemes = OrderedDict()          # {brick path below /recognizer: {scheme: value}}

        act = post_merge_activation if post_merge_activation is not None else _bricks.Tanh()
        post_merge_dims = [int(d) for d in post_merge_dims] if post_merge_dims else []
        if len(post_merge_dims) > 1:
            # Bias(d_1) -> act -> MLP([act] * (k-1) + [Identity()], [d_j // pieces] + [V]) (recognizer.py:305-320)
            k, pieces = len(post_merge_dims), int(getattr(act, "num_pieces", 1))
            if k > _lib.LVSR_MAX_READOUT:
                unsupported("a post-merge MLP of %d layers (post_merge_dims of at most %d entries)"
                            % (k, _lib.LVSR_MAX_READOUT))
            if any(d < 8 or d % 8 for d in post_merge_dims):
                raise ValueError("post_merge_dims %r: every width must be a positive multiple of 8" % (post_merge_dims,))
            if pieces > 1:
                # the reference's MLP takes d_j // pieces inputs and its Maxout divides them again: the graph fails
                raise ValueError("post_merge_dims %r under Maxout(%d): a Maxout of more than one piece takes one "
                                 "post-merge layer only" % (post_merge_dims, pieces))
            widest = _lib.load().lvsr_readout_max_width()
            if post_merge_dims[-1] > widest:
                unsupported("a last post-merge width of %d (at most %d: the widest the readout kernels stage in "
                            "shared memory)" % (post_merge_dims[-1], widest))
        if dim_matcher is None:
            dim_matcher = dim_dec                                  # recognizer.py:225-226
        content = attention_type == "content"
        if conv_n is None and not content:
            raise ValueError("conv_n is required for content_and_conv attention")
        subsample = list(subsample) if subsample else [1] * len(dims_bidir)
        prior = dict(prior) if prior else dict(type="expanding", initial_begin=0, initial_end=10000,
                                               min_speed=0, max_speed=0)    # lvsr/bricks/attention.py:72-74
        if content:
            # SequenceContentAttention takes no conv, normaliser or prior (lvsr/bricks/recognizer.py:261-265): the
            # reference ignores these keys, and so does the library
            conv_n, conv_num_filters, energy_normalizer, prior = 0, 0, None, None
        self.net = dict(
            num_features=int(input_dims["recordings"]), dims_bidir=[int(d) for d in dims_bidir],
            subsample=[int(k) for k in subsample], dim_dec=int(dim_dec), dim_matcher=int(dim_matcher),
            conv_n=int(conv_n), conv_num_filters=int(conv_num_filters), num_phonemes=int(num_phonemes),
            # LookupFeedback(V+1, dim) or OneOfNFeedback(V+1) whose feedback is the one-hot vector (recognizer.py:278-284)
            dim_feedback=(int(dim_dec if dim_output_embedding is None else dim_output_embedding) if embed_outputs
                          else int(num_phonemes) + 1),
            embed_outputs=bool(embed_outputs),
            post_merge_dim=post_merge_dims[0] if post_merge_dims else int(num_phonemes),
            post_merge_dims=post_merge_dims,
            post_merge_activation=act.kind, maxout_pieces=int(getattr(act, "num_pieces", 1)),
            use_states_for_readout=bool(use_states_for_readout),
            energy_normalizer=energy_normalizer or "softmax", prior=prior, attention_type=attention_type,
            dec_stack=int(dec_stack), bidir=bool(bidir))
        if bottom_dims:
            self.net["bottom"] = dict(dims=bottom_dims, activation=bottom_kind)
        if not post_merge_dims:
            # Readout's default post_merge is a bare Bias on readout_dim (sequence_generators.py:596-599)
            self.net["post_merge_activation"] = "identity"
            unsupported("readout without post_merge_dims")

        # brick-tree handles
        if content:
            attention = _Child("cont_att")
        else:
            attention = _Child("conv_att", prior=prior, energy_normalizer=self.net["energy_normalizer"])
        transition = _Child("att_trans", attention=attention)
        readout = _Child("readout", emitter=_Child("emitter"), readout=None)
        self.generator = _Child("generator", transition=transition, readout=readout)
        self.encoder = _Child("encoder")
        self.top = _Child("top")
        self.bottom = _Child("bottom")
        self.children = [self.encoder, self.top, self.bottom, self.generator]

        # named inputs of the reference's graphs (lvsr/bricks/recognizer.py:351-361)
        self.inputs = OrderedDict(recordings=_Variable("recordings"))
        self.single_inputs = OrderedDict(recordings=_Variable("recordings"))
        self.inputs_mask = _Variable("recordings_mask")
        self.labels = _Variable("labels")
        self.labels_mask = _Variable("labels_mask")
        self.single_labels = _Variable("labels")
        self.n_steps = _Variable("n_steps")

        self._device = device
        self._handle = None
        self._beam_search = None
        self.beam_size = None
        self._ctor_state = None

    # ------------------------------------------------------------------------------
    # handle / device
    # ------------------------------------------------------------------------------
    def _torch(self):
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError("attention-lvcsr_b200 needs a CUDA device (no CPU fallback)")
        return torch

    @property
    def device(self):
        torch = self._torch()
        if self._device is None:
            self._device = torch.device("cuda", torch.cuda.current_device())
        return torch.device(self._device)

    def _make_config(self):
        import ctypes as C
        n = self.net
        cfg = _lib.LvsrConfig()
        cfg.num_features = n["num_features"]
        cfg.num_layers = len(n["dims_bidir"])
        for i, (d, k) in enumerate(zip(n["dims_bidir"], n["subsample"])):
            cfg.dims_bidir[i] = d
            cfg.subsample[i] = k
        cfg.dim_dec = n["dim_dec"]
        cfg.dim_matcher = n["dim_matcher"]
        cfg.conv_n = n["conv_n"]
        cfg.conv_num_filters = n["conv_num_filters"]
        cfg.num_phonemes = n["num_phonemes"]
        cfg.dim_feedback = n["dim_feedback"]
        cfg.post_merge_dim = n["post_merge_dim"]
        cfg.maxout_pieces = n["maxout_pieces"]
        cfg.post_merge_activation = _lib.ACTIVATIONS[n["post_merge_activation"]]
        cfg.use_states_for_readout = int(n["use_states_for_readout"])
        cfg.energy_normalizer = _lib.NORMALIZERS[n["energy_normalizer"]]
        cfg.attention_type = _lib.ATTENTION_TYPES[n.get("attention_type", "content_and_conv")]
        p = n["prior"] or {}
        cfg.prior_type = _lib.PRIORS[p.get("type", "expanding")]
        cfg.prior_initial_begin = float(p.get("initial_begin", 0))
        cfg.prior_initial_end = float(p.get("initial_end", 10000))
        cfg.prior_min_speed = float(p.get("min_speed", 0))
        cfg.prior_max_speed = float(p.get("max_speed", 0))
        cfg.prior_before = float(p.get("before", 0))
        cfg.prior_after = float(p.get("after", 0))
        cfg.one_of_n_feedback = 0 if n.get("embed_outputs", True) else 1
        cfg.dec_stack = n.get("dec_stack", 1)
        return cfg

    def _make_bottom_config(self):
        """lvsr_bottom_config of the bottom MLP, None without one."""
        b = self.net.get("bottom")
        if not b:
            return None
        if len(b["dims"]) > _lib.LVSR_MAX_BOTTOM:
            raise NotImplementedError("attention-lvcsr_b200: a bottom MLP of %d layers (at most %d)"
                                      % (len(b["dims"]), _lib.LVSR_MAX_BOTTOM))
        out = _lib.LvsrBottomConfig()
        out.num_layers = len(b["dims"])
        for i, d in enumerate(b["dims"]):
            out.dims[i] = d
        out.activation = _lib.BOTTOM_ACTIVATIONS[b["activation"]]
        return out

    def _make_readout_config(self):
        """lvsr_readout_config of a post-merge MLP deeper than one layer, None otherwise."""
        dims = self.net.get("post_merge_dims") or []
        if len(dims) <= 1:
            return None
        out = _lib.LvsrReadoutConfig()
        out.num_layers = len(dims)
        for i, d in enumerate(dims):
            out.dims[i] = d
        return out

    def _require_ready(self):
        if self._handle is None:
            import ctypes as C
            torch = self._torch()
            lib = _lib.load()
            with torch.cuda.device(self.device):
                h = C.c_void_p()
                cfg = self._make_config()
                bottom = self._make_bottom_config()
                readout = self._make_readout_config()
                if readout is not None:
                    _lib.check(lib.lvsr_model_create_readout(C.byref(cfg), None if bottom is None else C.byref(bottom),
                                                             int(self.bidir), C.byref(readout), C.byref(h)))
                elif not self.bidir:
                    _lib.check(lib.lvsr_model_create_encoder(C.byref(cfg), None if bottom is None else C.byref(bottom),
                                                             0, C.byref(h)))
                elif bottom is None:
                    _lib.check(lib.lvsr_model_create(C.byref(cfg), C.byref(h)))
                else:
                    _lib.check(lib.lvsr_model_create_bottom(C.byref(cfg), C.byref(bottom), C.byref(h)))
            self._handle = h
            if self.lm:
                self._attach_lm(lib, h)
            if self.tle:
                self._set_criterion(lib, h)
        return self._handle

    @property
    def tle(self):
        """Task loss estimation (criterion mse_gain / mse_reward): RewardRegressionEmitter in place of SoftmaxEmitter."""
        return self.criterion["name"] != "log_likelihood"

    def _set_criterion(self, lib, h):
        """RewardRegressionEmitter(criterion, eos_label, num_phonemes, min_reward) (lvsr/bricks/recognizer.py:291-295),
        whose initial output is 0 (lvsr/bricks/__init__.py:198-201)."""
        import ctypes as C
        crit = _lib.LvsrCriterion(name=_lib.CRITERIA[self.criterion["name"]], eos_label=int(self.eos_label),
                                  initial_output=0, min_reward=float(self.criterion.get("min_reward", -1.0)))
        try:
            _lib.check(lib.lvsr_model_set_criterion(h, C.byref(crit)))
        except Exception:
            lib.lvsr_model_destroy(h)
            self._handle = None
            raise

    def _attach_lm(self, lib, h):
        """LanguageModel + ShallowFusionReadout (lvsr/bricks/recognizer.py:322-338) on the handle."""
        import ctypes as C
        t, o = self._lm_tables, self.lm
        fusion = _lib.LvsrLmFusion(weight=float(o["weight"]), am_beta=float(o["am_beta"]),
                                   no_transition_cost=float(o["no_transition_cost"]),
                                   normalize_am_weights=int(bool(o["normalize_am_weights"])),
                                   normalize_lm_weights=int(bool(o["normalize_lm_weights"])),
                                   normalize_tot_weights=int(bool(o["normalize_tot_weights"])))
        try:
            _lib.check(lib.lvsr_model_set_lm(h, t["num_states"], t["start"], t["offsets"].ctypes.data, len(t["label"]),
                                             t["label"].ctypes.data, t["next"].ctypes.data, t["weight"].ctypes.data,
                                             C.byref(fusion)))
        except Exception:
            lib.lvsr_model_destroy(h)
            self._handle = None
            raise

    def __del__(self):
        try:
            if self._handle is not None:
                _lib.load().lvsr_model_destroy(self._handle)
                self._handle = None
        except Exception:
            pass

    def _stream(self):
        return self._torch().cuda.current_stream(self.device).cuda_stream

    # ------------------------------------------------------------------------------
    # parameters
    # ------------------------------------------------------------------------------
    def parameter_shapes(self):
        import ctypes as C
        lib, h = _lib.load(), self._require_ready()
        out = OrderedDict()
        for i in range(lib.lvsr_model_num_params(h)):
            shape = (C.c_int64 * 2)()
            ndim = C.c_int32()
            _lib.check(lib.lvsr_model_param_shape(h, i, shape, C.byref(ndim)))
            out[lib.lvsr_model_param_name(h, i).decode()] = tuple(int(shape[j]) for j in range(ndim.value))
        return out

    def set_parameter_values(self, values):
        """Model.set_parameter_values: {Blocks parameter path: ndarray}."""
        lib, h = _lib.load(), self._require_ready()
        shapes = self.parameter_shapes()
        for name, value in values.items():
            if name not in shapes:
                raise KeyError("unknown parameter %s" % name)
            arr = np.ascontiguousarray(value, dtype=np.float32)
            if tuple(arr.shape) != shapes[name]:
                raise ValueError("parameter %s: expected shape %s, got %s" % (name, shapes[name], arr.shape))
            _lib.check(lib.lvsr_model_set_param(h, name.encode(), arr.ctypes.data, arr.size))
        _lib.check(lib.lvsr_model_finalize(h))

    def get_parameter_values(self):
        lib, h = _lib.load(), self._require_ready()
        out = OrderedDict()
        for name, shape in self.parameter_shapes().items():
            arr = np.empty(shape, dtype=np.float32)
            _lib.check(lib.lvsr_model_get_param(h, name.encode(), arr.ctypes.data, arr.size))
            out[name] = arr
        return out

    _ROOT_SCHEMES = ("weights_init", "biases_init", "rec_weights_init", "initial_states_init")
    _BRICK_SCHEMES = ("weights_init", "biases_init")

    def set_initialization(self, path, **schemes):
        """Initialisation schemes of the Blocks brick at `path`, as one entry of config['initialization'] sets them
        (lvsr/main.py:223-231).  '/recognizer' takes the four schemes of the recognizer itself; a deeper path takes
        weights_init / biases_init, which initialize() applies to the parameters of that brick and of the bricks
        below it, overriding every shallower path's.  A path naming no brick of the model is refused by initialize().
        """
        root = "/" + self.name
        allowed = self._ROOT_SCHEMES if path == root else self._BRICK_SCHEMES
        unknown = sorted(set(schemes) - set(allowed))
        if unknown:
            raise TypeError("initialization of %s: %s not supported (only %s)" % (path, unknown, ", ".join(allowed)))
        if path == root:
            for attr, value in schemes.items():
                setattr(self, attr, value)
        else:
            self._brick_schemes.setdefault(path, {}).update(schemes)

    def initial_values(self, shapes, seed=1):
        """The values initialize() sets, for the parameters `shapes` ({Blocks name: shape} in brick order):
        Blocks ``initialize()`` with one RandomState walked in brick order; a recurrent brick takes
        rec_weights_init for all three matrices, initial states take initial_states_init
        (lvsr/bricks/recognizer.py:363-373; B/bricks/recurrent.py:568-580).  The schemes of set_initialization's
        deeper paths are pushed after those of /recognizer (lvsr/main.py:223-231, sorted by depth), so the deepest
        path holding a parameter's brick decides that parameter's scheme.  Such a push sets weights_init only, so
        under it a recurrent brick's gate matrices follow the path while state_to_state keeps rec_weights_init
        (its recurrent_weights_init) when /recognizer sets one."""
        w_init = self.weights_init or _bricks.IsotropicGaussian(0.01)
        b_init = self.biases_init or _bricks.Constant(0.0)
        rec_init = self.rec_weights_init or w_init
        h0_init = self.initial_states_init or _bricks.Constant(0.0)
        overrides = self._brick_schemes
        bricks = set()
        for name in shapes:
            parts = name.rsplit(".", 1)[0].split("/")
            bricks.update("/".join(parts[:i]) for i in range(2, len(parts) + 1))
        for path in overrides:
            if path not in bricks:
                # the reference's `brick, = Selector(recognizer).select(path).bricks` finds no brick
                raise ValueError("initialization: no brick of the model at %s" % path)

        def scheme(name, attr, default):
            brick = name.rsplit(".", 1)[0]
            holders = [p for p, s in overrides.items() if attr in s and (brick == p or brick.startswith(p + "/"))]
            return overrides[max(holders, key=lambda p: p.count("/"))][attr] if holders else default

        rng = np.random.RandomState(seed)
        values = OrderedDict()
        for name, shape in shapes.items():
            leaf = name.rsplit(".", 1)[1]
            if leaf == "b":
                v = scheme(name, "biases_init", b_init).generate(rng, shape)
            elif leaf == "state_to_state":
                v = (self.rec_weights_init or scheme(name, "weights_init", w_init)).generate(rng, shape)
            elif leaf == "state_to_gates":
                d = shape[0]
                init = scheme(name, "weights_init", rec_init)
                v = np.hstack([init.generate(rng, (d, d)), init.generate(rng, (d, d))])
            elif leaf == "initial_state":
                v = h0_init.generate(rng, shape)
            else:
                v = scheme(name, "weights_init", w_init).generate(rng, shape)
            values[name] = np.asarray(v, dtype=np.float32).reshape(shape)
        return values

    def initialize(self, seed=1):
        """Blocks ``initialize()``: the parameters become initial_values(parameter_shapes(), seed)."""
        self.set_parameter_values(self.initial_values(self.parameter_shapes(), seed))

    def load_params(self, path):
        """Blocks checkpoint (tar with a ``_parameters`` npz whose keys use '|' for '/':
        libs/blocks/blocks/serialization.py:264-282,606-610) or a plain .npz.  Like
        Model.set_parameter_values (libs/blocks/blocks/model.py:120-146) unknown names and missing parameters
        are LOGGED, not raised; missing parameters keep their current values."""
        values = self.load_checkpoint_values(path)
        shapes = self.parameter_shapes()
        unknown = sorted(set(values) - set(shapes))
        missing = sorted(set(shapes) - set(values))
        if unknown:
            logger.error("unknown parameter names: {}\n".format(unknown))
        if missing:
            logger.error("missing values for parameters: {}\n".format(missing))
        self.set_parameter_values({k: v for k, v in values.items() if k in shapes})
        return dict(unknown=unknown, missing=missing)

    @staticmethod
    def load_checkpoint_values(path):
        """{Blocks parameter name: array} of a checkpoint load_params reads, every name it holds."""
        if tarfile.is_tarfile(path):
            with tarfile.open(path) as tar:
                data = np.load(io.BytesIO(tar.extractfile("_parameters").read()))
        else:
            data = np.load(path)
        return {k.replace("|", "/"): data[k] for k in data.files}

    def save_params(self, path, extra=None):
        """Write the parameters the way blocks.serialization.dump stores them separately: a tar archive with one
        member ``_parameters`` = numpy.savez of {brick path with '|' for '/': array}
        (libs/blocks/blocks/serialization.py:136,264-282,493-500,606-610) -- readable by the reference's
        load_parameters and by load_params above.  ``extra``: more {Blocks name: array} of the same model, such as
        the adaptive-noise parameters of GradientDescent.noise_parameter_values()."""
        values = OrderedDict(self.get_parameter_values())
        values.update(extra or {})
        buf = io.BytesIO()
        np.savez(buf, **{k.replace("/", "|"): v for k, v in values.items()})
        payload = buf.getvalue()
        with tarfile.open(path, "w") as tar:
            info = tarfile.TarInfo("_parameters")
            info.size = len(payload)
            tar.addfile(info, io.BytesIO(payload))

    # pickling: device handles do not travel (lvsr/bricks/recognizer.py:549-562 drops the compiled functions)
    def __getstate__(self):
        state = dict(self.__dict__)
        for attr in ("_handle", "_beam_search", "_generator_state", "_lm_tables"):    # the FST reloads from lm['path']
            state.pop(attr, None)
        state["_device"] = None if self._device is None else str(self._device)
        state["_saved_parameters"] = None if self._handle is None else self.get_parameter_values()
        return state

    def __setstate__(self, state):
        saved = state.pop("_saved_parameters", None)
        self.__dict__.update(state)
        self._handle = None
        self._beam_search = None
        lm = self.__dict__.get("lm")
        self.lm = lm
        self._lm_tables = _lm.load(lm["path"], self.character_map, self.net["num_phonemes"]) if lm else None
        if saved is not None:
            try:
                self.set_parameter_values(saved)
            except RuntimeError:           # unpickled where no GPU is visible: parameters stay on the host copy
                self._pending_parameters = saved

    # ------------------------------------------------------------------------------
    # device-side operators (torch tensors in, torch tensors out)
    # ------------------------------------------------------------------------------
    def _dev(self, a, dtype=None):
        torch = self._torch()
        if a is None:
            return None
        if isinstance(a, torch.Tensor):
            t = a.to(self.device)
        else:
            t = torch.as_tensor(np.ascontiguousarray(a), device=self.device)
        if dtype is not None and t.dtype != dtype:
            t = t.to(dtype)
        return t.contiguous()

    def launch_status(self):
        """(status, stepwise_fallbacks) of the persistent decoder (lvsr_model_status): status 0 = the last
        cost_matrix launch completed; the counter says how often a failed launch was re-run step-wise."""
        import ctypes as C
        lib, h = _lib.load(), self._require_ready()
        st, fb = C.c_int32(), C.c_int64()
        _lib.check(lib.lvsr_model_status(h, C.byref(st), C.byref(fb)))
        return int(st.value), int(fb.value)

    def decoder_plan(self):
        """Plan of the last cost_matrix (lvsr_model_decoder_plan) as a dict: ran (the persistent decoder ran),
        kernel ("dec_scan", "dec_scan<COMPACT>", "dec_content" or "stepwise"), cs, grid, nisl, nrg, ncg, nc1, nc2,
        nc3, tc_cap, wh_rows, red_alias, max_clusters (the planner's last occupancy answer), att_cs (cluster
        size of the last attention step) and l2_evict_first_kb (KB of P and H per step loaded L2 evict-first; 0: none)."""
        import ctypes as C
        lib, h = _lib.load(), self._require_ready()
        out = (C.c_int32 * 16)()
        _lib.check(lib.lvsr_model_decoder_plan(h, out))
        plan = {k: int(out[i]) for i, k in enumerate(_lib.PLAN_SLOTS)}
        plan["ran"] = bool(plan["ran"])
        plan["kernel"] = _lib.PLAN_KERNELS[plan["kernel"]]
        return plan

    def _encoder_plan_row(self, layer):
        import ctypes as C
        lib, h = _lib.load(), self._require_ready()
        out = (C.c_int32 * 16)()
        _lib.check(lib.lvsr_model_encoder_plan(h, int(layer), out))
        plan = {k: int(out[i]) for i, k in enumerate(_lib.ENC_PLAN_SLOTS)}
        for k in ("proj", "wgrad", "dx"):
            plan[k] = _lib.ENC_PATHS[plan[k]]
        plan["bigru"] = _lib.ENC_BIGRU_KERNELS[plan["bigru"]]
        plan["operands"] = _lib.ENC_OPERANDS[plan["operands"]]
        plan["tape"] = bool(plan["tape"])
        if layer >= 0:
            ov = (C.c_int32 * 3)()
            _lib.check(lib.lvsr_model_encoder_overlap(h, int(layer), ov))
            plan["overlap"], plan["tiles_beside"], plan["tiles_after"] = bool(ov[0]), int(ov[1]), int(ov[2])
        return plan

    def encoder_overlap_claims(self, layer, tiles):
        """lvsr_model_encoder_overlap_claims: int32 [tiles, 3], row c = (m-tile + 1, forward and backward scan progress)
        at which the projection of `layer` claimed its tile c beside the previous scan (zeros: done after the scan)."""
        import ctypes as C
        import numpy as np
        lib, h = _lib.load(), self._require_ready()
        out = np.zeros((int(tiles), 3), dtype=np.int32)
        _lib.check(lib.lvsr_model_encoder_overlap_claims(h, int(layer), out.ctypes.data_as(C.POINTER(C.c_int32)),
                                                         out.size))
        return out

    def encoder_plan(self):
        """What the encoder ran (lvsr_model_encoder_plan), one dict per layer.  Of the last encoder forward: proj (fork
        projection GEMM: "tc" or "ffma"), kpad (its contraction as the tensor-core GEMM stores it, 0 on FFMA), operands
        (of that tensor-core GEMM: "f16x3" when the contraction is a multiple of 64, else "tf32x3"; None on FFMA), bigru
        ("mma" or "ffma"), tape (a training forward), rb and cs (rows and CTAs per cluster), clusters, resident (clusters
        of that kernel the device holds at once), waves and T (frames scanned); overlap (the projection ran beside the
        previous layer's scan, lvsr_model_encoder_overlap), tiles_beside and tiles_after (its output tiles computed
        beside that scan and after it).  Of the last training step: bwd_cs (CTAs per cluster of the reverse-time scan),
        wgrad ("tc" or "ffma"), wgrad_splits, wgrad_kpad (the padded contraction over T*B rows, 0 on FFMA) and dx ("tc",
        "ffma", or None for layer 0 without a bottom MLP).  None / 0: not run."""
        return [self._encoder_plan_row(l) for l in range(len(self.net["dims_bidir"]))]

    def preprocess_plan(self):
        """Path of the last preprocess GEMM (lvsr_model_encoder_plan, layer -1): {"proj": "tc" | "ffma", "kpad": ...}."""
        plan = self._encoder_plan_row(-1)
        return {"proj": plan["proj"], "kpad": plan["kpad"]}

    def encoded_length(self, T):
        return int(_lib.load().lvsr_encoded_length(self._require_ready(), int(T)))

    @property
    def bidir(self):
        """net.bidir: Bidirectional encoder layers (True) or forward-only ones (False)."""
        return self.net.get("bidir", True)

    @property
    def dim_encoded(self):
        """Width of the encoded frames: both directions' states of the last layer, or its one direction's."""
        return (2 if self.bidir else 1) * self.net["dims_bidir"][-1]

    @property
    def dim_state(self):
        """Floats of a decoder state row: dim_dec, or with dec_stack 2 the states of both layers [s0 | s1]
        (the reference's "states" and "states#1")."""
        return self.net.get("dec_stack", 1) * self.net["dim_dec"]

    def encode(self, recordings, recordings_mask=None):
        """Encoder.apply (lvsr/bricks/__init__.py:71-78): [T,B,F], [T,B] -> ([T',B,E], [T',B])."""
        torch = self._torch()
        lib, h = _lib.load(), self._require_ready()
        x = self._dev(recordings, torch.float32)
        m = self._dev(recordings_mask, torch.float32)
        if x.dim() != 3:
            raise ValueError("encode: recordings [T,B,F] expected")
        T, B, F = x.shape
        if F != self.net["num_features"]:
            raise ValueError("expected %d features, got %d" % (self.net["num_features"], F))
        if m is not None and tuple(m.shape) != (T, B):
            raise ValueError("encode: recordings_mask must be [%d, %d], got %s" % (T, B, tuple(m.shape)))
        Tp = self.encoded_length(T)
        att = torch.empty((Tp, B, self.dim_encoded), dtype=torch.float32, device=self.device)
        attm = torch.empty((Tp, B), dtype=torch.float32, device=self.device)
        _lib.check(lib.lvsr_encoder_forward(h, _ptr(x), _ptr(m), T, B, _ptr(att), _ptr(attm), self._stream()))
        return att, attm

    def preprocess(self, attended):
        torch = self._torch()
        lib, h = _lib.load(), self._require_ready()
        Tp, U, _ = attended.shape
        out = torch.empty((Tp, U, self.net["dim_matcher"]), dtype=torch.float32, device=self.device)
        _lib.check(lib.lvsr_preprocess(h, _ptr(attended), Tp, U, _ptr(out), self._stream()))
        return out

    def _check_labels(self, labels):
        """Theano's lookup raises IndexError on a symbol outside the table; host arrays are
        checked here (device tensors are the caller's contract: no hidden synchronisation)."""
        if isinstance(labels, np.ndarray) and labels.size:
            lo, hi = int(labels.min()), int(labels.max())
            if lo < 0 or hi >= self.net["num_phonemes"]:
                raise ValueError("labels must lie in [0, %d): got %d..%d" % (self.net["num_phonemes"], lo, hi))

    def cost_matrix(self, labels, labels_mask, attended, attended_mask, return_all=False, groundtruth=None):
        """generator.cost_matrix (B/bricks/sequence_generators.py:319-326) on device tensors.  Under task loss
        estimation the labels are scored against ``groundtruth`` [Lg, B] (None: the labels themselves), as
        get_cost_graph substitutes it (recognizer.py:423-450); log-likelihood ignores it."""
        torch = self._torch()
        lib, h = _lib.load(), self._require_ready()
        self._check_labels(labels)
        y = self._dev(labels, torch.int64)
        ym = self._dev(labels_mask, torch.float32)
        att = self._dev(attended, torch.float32)
        attm = self._dev(attended_mask, torch.float32)
        if y.dim() != 2 or att.dim() != 3 or attm.dim() != 2:
            raise ValueError("cost_matrix: labels [L,B], attended [T',B,E], attended_mask [T',B] expected")
        L, B = y.shape
        Tp = att.shape[0]
        if L < 1 or B < 1 or Tp < 1:
            raise ValueError("cost_matrix: empty labels or attended sequence")
        if tuple(att.shape) != (Tp, B, self.dim_encoded):
            raise ValueError("cost_matrix: attended must be [%d, %d, %d], got %s" % (Tp, B, self.dim_encoded, tuple(att.shape)))
        if tuple(attm.shape) != (Tp, B):
            raise ValueError("cost_matrix: attended_mask must be [%d, %d], got %s" % (Tp, B, tuple(attm.shape)))
        if ym is not None and tuple(ym.shape) != (L, B):
            raise ValueError("cost_matrix: labels_mask must be [%d, %d], got %s" % (L, B, tuple(ym.shape)))
        g = None
        if groundtruth is not None and self.tle:
            self._check_labels(groundtruth)
            g = self._dev(groundtruth, torch.int64)
            if g.dim() != 2 or g.shape[1] != B or g.shape[0] < 1:
                raise ValueError("cost_matrix: groundtruth must be [Lg, %d], got %s" % (B, tuple(g.shape)))
        costs = torch.empty((L, B), dtype=torch.float32, device=self.device)
        extra = {}
        if return_all:
            extra = dict(weights=torch.empty((L, B, Tp), dtype=torch.float32, device=self.device),
                         energies=torch.empty((L, B, Tp), dtype=torch.float32, device=self.device),
                         states=torch.empty((L, B, self.dim_state), dtype=torch.float32, device=self.device),
                         weighted_averages=torch.empty((L, B, self.dim_encoded), dtype=torch.float32,
                                                       device=self.device))
        _lib.check(lib.lvsr_cost_matrix_groundtruth(
            h, _ptr(att), _ptr(attm), Tp, B, _ptr(y), _ptr(ym), L, _ptr(g), 0 if g is None else g.shape[0],
            _ptr(costs), _ptr(extra.get("weights")), _ptr(extra.get("energies")), _ptr(extra.get("states")),
            _ptr(extra.get("weighted_averages")), self._stream()))
        if return_all:
            extra["costs"] = costs
            return extra
        return costs

    def alignment_statistics(self, weights, labels_mask, out):
        """lvsr_alignment_stats: out[0] = sum of mask * sum_t w log(w + 1e-7), out[1] = the monotonicity penalty
        (lvsr/expressions.py:14-25) of weights [L,B,T'] on the device; out is a float64 device tensor of >= 2."""
        torch = self._torch()
        lib, h = _lib.load(), self._require_ready()
        L, B, Tp = weights.shape
        if weights.dtype != torch.float32 or not weights.is_contiguous():
            raise ValueError("alignment_statistics: contiguous float32 weights expected")
        if labels_mask is not None and (tuple(labels_mask.shape) != (L, B) or labels_mask.dtype != torch.float32):
            raise ValueError("alignment_statistics: labels_mask must be float32 [%d, %d]" % (L, B))
        if out.dtype != torch.float64 or out.numel() < 2:
            raise ValueError("alignment_statistics: out must be a float64 tensor of at least 2 elements")
        _lib.check(lib.lvsr_alignment_stats(h, _ptr(weights), _ptr(labels_mask), L, B, Tp, _ptr(out), self._stream()))
        return out

    def validation_statistics(self, recordings, recordings_mask, labels, labels_mask):
        """What one batch of the reference's validation (lvsr/main.py:550-568) accumulates: dict(cost = sum of the cost
        matrix, weights_entropy, weights_penalty (the sums of lvsr/expressions.py:14-25), num_labels = sum of the label
        mask, batch_size).  The encoder, the teacher-forced decoder with its alignment, and the statistics kernel run on
        device buffers; the results come back in one copy."""
        torch = self._torch()
        att, attm = self.encode(recordings, recordings_mask)
        self._check_labels(labels)
        y = self._dev(labels, torch.int64)
        ym = self._dev(labels_mask, torch.float32)
        L, B = y.shape
        # [entropy, penalty | costs [L, B] as float32]: one read-back
        buf = torch.empty((2 + (L * B + 1) // 2,), dtype=torch.float64, device=self.device)
        costs = buf[2:].view(torch.float32)[:L * B].view(L, B)
        weights = torch.empty((L, B, att.shape[0]), dtype=torch.float32, device=self.device)
        lib, h = _lib.load(), self._require_ready()
        if ym is not None and tuple(ym.shape) != (L, B):
            raise ValueError("validation_statistics: labels_mask must be [%d, %d], got %s" % (L, B, tuple(ym.shape)))
        _lib.check(lib.lvsr_cost_matrix(h, _ptr(att), _ptr(attm), att.shape[0], B, _ptr(y), _ptr(ym), L, _ptr(costs),
                                        _ptr(weights), None, None, None, self._stream()))
        self.alignment_statistics(weights, ym, buf)
        host = buf.cpu().numpy()
        host_costs = host[2:].view(np.float32)[:L * B]
        num_labels = float(L * B) if labels_mask is None else float(np.asarray(
            labels_mask.cpu() if isinstance(labels_mask, torch.Tensor) else labels_mask, dtype=np.float64).sum())
        return dict(cost=float(host_costs.astype(np.float64).sum()), weights_entropy=float(host[0]),
                    weights_penalty=float(host[1]), num_labels=num_labels, batch_size=int(B))

    # ------------------------------------------------------------------------------
    # reference-facing methods (numpy in, numpy out)
    # ------------------------------------------------------------------------------
    def cost(self, recordings, recordings_mask, labels, labels_mask):
        """SpeechRecognizer.cost (recognizer.py:375-390) through the host-buffer C entry
        point: copies in, encoder + teacher-forced decoder, costs [L, B] copied out."""
        lib, h = _lib.load(), self._require_ready()
        x = np.ascontiguousarray(recordings, dtype=np.float32)
        m = None if recordings_mask is None else np.ascontiguousarray(recordings_mask, dtype=np.float32)
        y = np.ascontiguousarray(labels, dtype=np.int64)
        self._check_labels(y)
        ym = None if labels_mask is None else np.ascontiguousarray(labels_mask, dtype=np.float32)
        if x.ndim != 3 or y.ndim != 2:
            raise ValueError("cost: recordings [T,B,F] and labels [L,B] expected")
        T, B, F = x.shape
        L = y.shape[0]
        if F != self.net["num_features"]:
            raise ValueError("expected %d features, got %d" % (self.net["num_features"], F))
        if T < 1 or B < 1 or L < 1:
            raise ValueError("cost: empty batch")
        if m is not None and m.shape != (T, B):
            raise ValueError("cost: recordings_mask must be [%d, %d], got %s" % (T, B, m.shape))
        if y.shape != (L, B):
            raise ValueError("cost: labels must be [L, %d], got %s" % (B, y.shape))
        if ym is not None and ym.shape != (L, B):
            raise ValueError("cost: labels_mask must be [%d, %d], got %s" % (L, B, ym.shape))
        costs = np.empty((L, B), dtype=np.float32)
        torch = self._torch()
        with torch.cuda.device(self.device):
            _lib.check(lib.lvsr_recognizer_cost_host(
                h, x.ctypes.data, None if m is None else m.ctypes.data, y.ctypes.data,
                None if ym is None else ym.ctypes.data, T, B, L, costs.ctypes.data, self._stream()))
        return costs

    def analyze(self, inputs, groundtruth, prediction=None):
        """recognizer.py:452-494: one utterance, mask of ones, no label mask.  Under task loss estimation the
        prediction is scored against the groundtruth."""
        rec = np.asarray(dict(inputs)["recordings"], dtype=np.float32)[:, None, :]
        labels = np.asarray(groundtruth if prediction is None else prediction, dtype=np.int64)[:, None]
        att, attm = self.encode(rec, np.ones(rec.shape[:2], dtype=np.float32))
        r = self.cost_matrix(labels, None, att, attm, return_all=True,
                             groundtruth=np.asarray(groundtruth, dtype=np.int64)[:, None])
        return [r["costs"][:, 0].cpu().numpy(), r["weights"][:, 0, :].cpu().numpy(),
                r["energies"][:, 0, :].cpu().numpy()]

    def init_beam_search(self, beam_size):
        """recognizer.py:496-511."""
        if self._beam_search is not None and self.beam_size == beam_size:
            return
        self.beam_size = beam_size
        self._beam_search = BeamSearch(beam_size, self)
        self._beam_search.compile()

    def beam_search(self, inputs, **kwargs):
        """recognizer.py:513-533: inputs {'recordings': [T, F]} -> (outputs, costs)."""
        self.init_beam_search(self.beam_size)
        inputs = dict(inputs)
        rec = np.asarray(inputs.pop("recordings"), dtype=np.float32)
        if inputs:
            raise Exception("Unknown inputs passed to beam search: {}".format(list(inputs.keys())))
        max_length = int(rec.shape[0] / self.max_decoded_length_scale)
        return self._beam_search.search({"recordings": rec[:, None, :]}, self.eos_label, max_length,
                                        ignore_first_eol=self.data_prepend_eos, **kwargs)

    def beam_search_many(self, inputs_list, **kwargs):
        """beam_search for a list of {'recordings': [T_u, F]} decoded together on the GPU (one set of launches per
        step for all utterances, BeamSearch.search_many); returns [(outputs, costs), ...] in order.  The
        reference decodes one utterance at a time (lvsr/main.py:806-821 loops over the data stream)."""
        self.init_beam_search(self.beam_size)
        recs = []
        for inputs in inputs_list:
            inputs = dict(inputs)
            recs.append(np.asarray(inputs.pop("recordings"), dtype=np.float32))
            if inputs:
                raise Exception("Unknown inputs passed to beam search: {}".format(list(inputs.keys())))
        max_lengths = [int(x.shape[0] / self.max_decoded_length_scale) for x in recs]
        return self._beam_search.search_many(recs, self.eos_label, max_lengths,
                                             ignore_first_eol=self.data_prepend_eos, **kwargs)

    # ---- generate / sample (B/bricks/sequence_generators.py:328-377; recognizer.py:535-547) ----
    def generate(self, recordings, recordings_mask=None, n_steps=None, sample=True, seed=None):
        """SequenceGenerator.generate iterated n_steps times for a batch [T,B,F]: glimpses -> readout -> emit ->
        feedback -> next state.  ``sample=True`` emits from the softmax like SoftmaxEmitter.emit
        (sequence_generators.py:772-778; a seeded Philox stream on the device instead of Theano's MRG stream, so
        draws differ from the reference while their distribution does not), ``sample=False`` emits the arg-max.
        Returns dict(outputs [n,B] int64, costs [n,B] = -log p(emitted), states [n,B,dim_state], weights [n,B,T']).
        Under task loss estimation RewardRegressionEmitter emits the arg-max of the readouts whatever ``sample`` says,
        and the costs are the emitted readouts (its cost, lvsr/bricks/__init__.py:185-192); with a language model
        these are the fused readouts, and the LM state of every row advances by its emitted symbol."""
        if self.lm and not self.tle:
            # LMEmitter.emit returns zeros in the reference: generating with an LM is not defined there
            raise NotImplementedError("attention-lvcsr_b200: generate / sample with a language model")
        torch = self._torch()
        att, attm = self.encode(recordings, recordings_mask)
        B, Tp = att.shape[1], att.shape[0]
        if n_steps is None:
            n_steps = int(np.asarray(recordings).shape[0] / self.max_decoded_length_scale)
        ctx = dict(attended=att, attended_mask=attm, preprocessed=self.preprocess(att))
        st = self._initial_states(Tp, B)
        if self.lm:
            st.update(self._lm_initial_states(B))
        gen = None
        if sample:
            gen = torch.Generator(device=self.device)
            gen.manual_seed(1 if seed is None else int(seed))
        outs, costs, states, weights = [], [], [], []
        for _ in range(int(n_steps)):
            neglogp = self._logprobs(ctx, st)
            if sample and not self.tle:
                y = torch.multinomial(torch.exp(-neglogp), 1, generator=gen)[:, 0]
            else:
                y = neglogp.argmin(dim=1)
            picked = neglogp.gather(1, y[:, None])[:, 0]
            costs.append(-picked if self.tle else picked)
            lm_st = self._lm_next_states(st, y) if self.lm else {}
            st = self._next_states(ctx, st, y)
            st.update(lm_st)
            outs.append(y)
            states.append(st["states"])
            weights.append(st["weights"])
        return dict(outputs=torch.stack(outs).cpu().numpy(), costs=torch.stack(costs).cpu().numpy(),
                    states=torch.stack(states).cpu().numpy(), weights=torch.stack(weights).cpu().numpy())

    def sample(self, inputs, n_steps=None, seed=None):
        """recognizer.py:540-547: one utterance {'recordings': [T,F]} -> sampled outputs [n_steps, 1]."""
        rec = np.asarray(dict(inputs)["recordings"], dtype=np.float32)[:, None, :]
        if n_steps is None:
            n_steps = int(rec.shape[0] / self.max_decoded_length_scale)
        return self.generate(rec, None, n_steps=n_steps, sample=True, seed=seed)["outputs"]

    def get_generate_graph(self, use_mask=True, n_steps=None):
        """recognizer.py:414-421 returns the symbolic generate application; here: a callable with the same inputs
        (recordings [, recordings_mask], n_steps) returning the dict of generate()."""
        def run(recordings, recordings_mask=None, n_steps=n_steps, **kw):
            return self.generate(recordings, recordings_mask if use_mask else None, n_steps=n_steps, **kw)
        return run

    def get_cost_graph(self, batch=True, prediction=None, prediction_mask=None):
        """recognizer.py:423-450: the cost 'graph' as a callable: batch=True takes (recordings, recordings_mask, labels,
        labels_mask) -> costs [L,B]; batch=False takes one utterance (recordings [T,F], labels [L]) -> costs [L]."""
        if batch:
            return lambda recordings, recordings_mask, labels, labels_mask: self.cost(recordings, recordings_mask, labels, labels_mask)
        return lambda recordings, labels: self.analyze({"recordings": recordings}, labels)[0]

    # ------------------------------------------------------------------------------
    # BeamSearch state functions (C-ABI calls)
    # ------------------------------------------------------------------------------
    def _initial_states(self, Tp, R):
        torch = self._torch()
        lib, h = _lib.load(), self._require_ready()
        dev = self.device
        st = OrderedDict(
            states=torch.empty((R, self.dim_state), dtype=torch.float32, device=dev),
            outputs=torch.empty((R,), dtype=torch.int64, device=dev),
            weighted_averages=torch.empty((R, self.dim_encoded), dtype=torch.float32, device=dev),
            weights=torch.empty((R, Tp), dtype=torch.float32, device=dev),
            energies=torch.empty((R, Tp), dtype=torch.float32, device=dev),
            step=torch.empty((R,), dtype=torch.int64, device=dev))
        _lib.check(lib.lvsr_initial_states(h, Tp, R, _ptr(st["states"]), _ptr(st["outputs"]),
                                           _ptr(st["weighted_averages"]), _ptr(st["weights"]),
                                           _ptr(st["energies"]), _ptr(st["step"]), self._stream()))
        return st

    # the language model's initial_state_computer / next_state_computer (FSTTransition, lvsr/bricks/language_models.py)
    def _lm_initial_states(self, R):
        torch = self._torch()
        lib, h = _lib.load(), self._require_ready()
        st = OrderedDict(lm_states=torch.empty((R, _lib.LM_MAX_STATES), dtype=torch.int32, device=self.device),
                         lm_weights=torch.empty((R, _lib.LM_MAX_STATES), dtype=torch.float64, device=self.device),
                         lm_add=torch.empty((R, self.net["num_phonemes"]), dtype=torch.float32, device=self.device))
        _lib.check(lib.lvsr_lm_initial_states(h, R, _ptr(st["lm_states"]), _ptr(st["lm_weights"]), _ptr(st["lm_add"]),
                                              self._stream()))
        return st

    def _lm_next_states(self, st, outputs):
        torch = self._torch()
        lib, h = _lib.load(), self._require_ready()
        y = self._dev(outputs, torch.int64)
        s, w = self._dev(st["lm_states"], torch.int32), self._dev(st["lm_weights"], torch.float64)
        R = s.shape[0]
        # the C ABI takes R rows of every array and no lengths: a short one would be read past its end
        if s.dim() != 2 or s.shape[1] != _lib.LM_MAX_STATES or tuple(w.shape) != tuple(s.shape) or tuple(y.shape) != (R,):
            raise ValueError("lm_next_states: states %s and weights %s must be [R, %d] and outputs %s [R]"
                             % (tuple(s.shape), tuple(w.shape), _lib.LM_MAX_STATES, tuple(y.shape)))
        nxt = OrderedDict(lm_states=torch.empty_like(s), lm_weights=torch.empty_like(w),
                          lm_add=torch.empty((R, self.net["num_phonemes"]), dtype=torch.float32, device=self.device))
        _lib.check(lib.lvsr_lm_next_states(h, R, _ptr(s), _ptr(w), _ptr(y), _ptr(nxt["lm_states"]),
                                           _ptr(nxt["lm_weights"]), _ptr(nxt["lm_add"]), self._stream()))
        return nxt

    def _row_utt(self, contexts, R):
        torch = self._torch()
        U = contexts["attended"].shape[1]
        ru = contexts.get("row_utt")
        if ru is None:
            if U == R:
                return None
            if U != 1:
                raise ValueError("contexts hold %d utterances for %d rows: pass row_utt" % (U, R))
            ru = torch.zeros((R,), dtype=torch.int32, device=self.device)
        return self._dev(ru, torch.int32)

    def _logprobs(self, contexts, st):
        """The emitter costs [R, V] of the rows of st; fused with the language model when st carries its cost rows
        (``lm_add``, from _lm_initial_states / _lm_next_states)."""
        torch = self._torch()
        lib, h = _lib.load(), self._require_ready()
        att = contexts["attended"]
        Tp, U, _ = att.shape
        R = st["states"].shape[0]
        ru = self._row_utt(contexts, R)
        V = self.net["num_phonemes"]
        out = torch.empty((R, V), dtype=torch.float32, device=self.device)
        lm_add = st.get("lm_add")
        if lm_add is not None:
            lm_add = self._dev(lm_add, torch.float32)
            if tuple(lm_add.shape) != (R, V):      # the C ABI reads R rows of V
                raise ValueError("logprobs: lm_add must be [%d, %d], got %s" % (R, V, tuple(lm_add.shape)))
        _lib.check(lib.lvsr_logprobs_lm(h, _ptr(att), _ptr(contexts.get("preprocessed")), _ptr(contexts["attended_mask"]),
                                        Tp, U, _ptr(ru), R, _ptr(st["states"].contiguous()),
                                        _ptr(st["weights"].contiguous()), _ptr(st["step"].contiguous()), _ptr(lm_add),
                                        _ptr(out), self._stream()))
        return out

    def _next_states(self, contexts, st, outputs):
        torch = self._torch()
        lib, h = _lib.load(), self._require_ready()
        att = contexts["attended"]
        Tp, U, _ = att.shape
        R = st["states"].shape[0]
        ru = self._row_utt(contexts, R)
        y = self._dev(outputs, torch.int64)
        nxt = OrderedDict(
            states=torch.empty_like(st["states"]), outputs=y,
            weighted_averages=torch.empty((R, self.dim_encoded), dtype=torch.float32, device=self.device),
            weights=torch.empty((R, Tp), dtype=torch.float32, device=self.device),
            energies=torch.empty((R, Tp), dtype=torch.float32, device=self.device),
            step=torch.empty((R,), dtype=torch.int64, device=self.device))
        _lib.check(lib.lvsr_next_states(
            h, _ptr(att), _ptr(contexts.get("preprocessed")), _ptr(contexts["attended_mask"]), Tp, U, _ptr(ru), R,
            _ptr(st["states"].contiguous()), _ptr(st["weights"].contiguous()), _ptr(st["step"].contiguous()),
            _ptr(y), _ptr(nxt["states"]), _ptr(nxt["weighted_averages"]), _ptr(nxt["weights"]),
            _ptr(nxt["energies"]), _ptr(nxt["step"]), self._stream()))
        return nxt
