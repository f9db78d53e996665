"""ctypes binding of csrc/liblvsr_b200.so -- the C ABI declared in include/lvsr_b200.h.

There is NO fallback: if the shared library is missing, importing the package works
(so host-only logic can be unit-tested) but any compute call raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# LVSR_B200_LIB: load another build of the same library (A/B measurements of kernel variants on one box)
LIB_PATH = os.environ.get("LVSR_B200_LIB") or os.path.join(_HERE, "csrc", "liblvsr_b200.so")

LVSR_MAX_LAYERS = 8
NORMALIZERS = {"softmax": 0, "logistic": 1, "relu": 2}
ACTIVATIONS = {"maxout": 0, "relu": 1, "tanh": 2, "identity": 3}
PRIORS = {"expanding": 0, "window_around_mean": 1, "window_around_median": 2}
ATTENTION_TYPES = {"content_and_conv": 0, "content": 1}
# slots of lvsr_model_decoder_plan's report (LVSR_PLAN_*) and the kernel names of its `kernel` slot (LVSR_PLAN_DEC_*)
PLAN_SLOTS = ("ran", "kernel", "cs", "grid", "nisl", "nrg", "ncg", "nc1", "nc2", "nc3", "tc_cap", "wh_rows", "red_alias",
              "att_cs", "max_clusters", "l2_evict_first_kb")
PLAN_KERNELS = ("stepwise", "dec_scan", "dec_scan<COMPACT>", "dec_content")
# slots of lvsr_model_encoder_plan's report (LVSR_ENC_*), the GEMM paths (LVSR_ENC_PATH_*), the operands of the
# tensor-core projection (LVSR_ENC_OPS_*) and the scan kernels (LVSR_ENC_BIGRU_*)
ENC_PLAN_SLOTS = ("proj", "kpad", "bigru", "tape", "rb", "cs", "clusters", "resident", "waves", "T", "bwd_cs", "wgrad",
                  "wgrad_splits", "wgrad_kpad", "dx", "operands")
ENC_PATHS = (None, "tc", "ffma")
ENC_OPERANDS = (None, "tf32x3", "f16x3")
ENC_BIGRU_KERNELS = (None, "ffma", "mma")


class LvsrConfig(C.Structure):
    """Mirror of ``lvsr_config`` (include/lvsr_b200.h)."""
    _fields_ = [
        ("num_features", C.c_int32),
        ("num_layers", C.c_int32),
        ("dims_bidir", C.c_int32 * LVSR_MAX_LAYERS),
        ("subsample", C.c_int32 * LVSR_MAX_LAYERS),
        ("dim_dec", C.c_int32),
        ("dim_matcher", C.c_int32),
        ("conv_n", C.c_int32),
        ("conv_num_filters", C.c_int32),
        ("num_phonemes", C.c_int32),
        ("dim_feedback", C.c_int32),
        ("post_merge_dim", C.c_int32),
        ("maxout_pieces", C.c_int32),
        ("post_merge_activation", C.c_int32),
        ("use_states_for_readout", C.c_int32),
        ("energy_normalizer", C.c_int32),
        ("prior_type", C.c_int32),
        ("prior_initial_begin", C.c_double),
        ("prior_initial_end", C.c_double),
        ("prior_min_speed", C.c_double),
        ("prior_max_speed", C.c_double),
        ("prior_before", C.c_double),
        ("prior_after", C.c_double),
        ("one_of_n_feedback", C.c_int32),
        ("attention_type", C.c_int32),
        ("dec_stack", C.c_int32),
    ]


LVSR_MAX_BOTTOM = 4
LVSR_MAX_READOUT = 4


class LvsrReadoutConfig(C.Structure):
    """Mirror of ``lvsr_readout_config`` (include/lvsr_b200.h)."""
    _fields_ = [("num_layers", C.c_int32), ("dims", C.c_int32 * LVSR_MAX_READOUT)]

LVSR_MAX_BOTTOM_DIM = 4096
# activations of the bottom MLP (LVSR_ACT_* values of lvsr_bottom_config.activation)
BOTTOM_ACTIVATIONS = {"relu": 1, "tanh": 2}


class LvsrBottomConfig(C.Structure):
    """Mirror of ``lvsr_bottom_config`` (include/lvsr_b200.h)."""
    _fields_ = [("num_layers", C.c_int32), ("dims", C.c_int32 * LVSR_MAX_BOTTOM), ("activation", C.c_int32)]


class LvsrTrainConfig(C.Structure):
    """Mirror of ``lvsr_train_config`` (include/lvsr_b200.h)."""
    _fields_ = [("gradient_threshold", C.c_float), ("use_momentum", C.c_int32), ("scale", C.c_float),
                ("momentum", C.c_float), ("use_adadelta", C.c_int32), ("decay_rate", C.c_float),
                ("epsilon", C.c_float), ("max_norm", C.c_float), ("burn_in_steps", C.c_int32), ("decay", C.c_float)]


class LvsrAdaptiveNoise(C.Structure):
    """Mirror of ``lvsr_adaptive_noise`` (include/lvsr_b200.h)."""
    _fields_ = [("init_sigma", C.c_double), ("model_cost_coefficient", C.c_double), ("num_examples", C.c_int64),
                ("seed", C.c_uint64)]


class LvsrAdaptiveClipping(C.Structure):
    """Mirror of ``lvsr_adaptive_clipping`` (include/lvsr_b200.h)."""
    _fields_ = [("initial_threshold", C.c_double), ("decay_rate", C.c_double), ("burnin_period", C.c_int32)]


class LvsrRegularization(C.Structure):
    """Mirror of ``lvsr_regularization`` (include/lvsr_b200.h)."""
    _fields_ = [("dropout", C.c_int32), ("noise_level", C.c_double), ("penalty_coof", C.c_double), ("seed", C.c_uint64)]


# slots of lvsr_train_noise_stats (LVSR_NOISE_*), under the reference's monitor names (lvsr/main.py:440-460)
NOISE_STATS = ("model_cost", "model_prior_mean", "model_prior_variance")

LM_MAX_STATES = 7


class LvsrLmFusion(C.Structure):
    """Mirror of ``lvsr_lm_fusion`` (include/lvsr_b200.h)."""
    _fields_ = [("weight", C.c_double), ("am_beta", C.c_double), ("no_transition_cost", C.c_double),
                ("normalize_am_weights", C.c_int32), ("normalize_lm_weights", C.c_int32),
                ("normalize_tot_weights", C.c_int32)]


# name of lvsr_criterion (LVSR_CRITERION_*)
CRITERIA = {"log_likelihood": 0, "mse_gain": 1, "mse_reward": 2}


class LvsrCriterion(C.Structure):
    """Mirror of ``lvsr_criterion`` (include/lvsr_b200.h)."""
    _fields_ = [("name", C.c_int32), ("eos_label", C.c_int32), ("initial_output", C.c_int32),
                ("min_reward", C.c_double)]


# window_type of lvsr_fbank_options (LVSR_WINDOW_*)
WINDOW_TYPES = {"povey": 0, "hamming": 1, "hanning": 2, "rectangular": 3}


class LvsrFbankOptions(C.Structure):
    """Mirror of ``lvsr_fbank_options`` (include/lvsr_b200.h)."""
    _fields_ = [("sample_frequency", C.c_double), ("frame_length", C.c_double), ("frame_shift", C.c_double),
                ("dither", C.c_double), ("preemphasis_coefficient", C.c_double), ("low_freq", C.c_double),
                ("high_freq", C.c_double), ("energy_floor", C.c_double), ("vtln_warp", C.c_double),
                ("seed", C.c_uint64), ("remove_dc_offset", C.c_int32), ("window_type", C.c_int32),
                ("round_to_power_of_two", C.c_int32), ("snip_edges", C.c_int32), ("num_mel_bins", C.c_int32),
                ("use_energy", C.c_int32), ("raw_energy", C.c_int32), ("use_log_fbank", C.c_int32),
                ("use_power", C.c_int32), ("htk_compat", C.c_int32), ("delta_order", C.c_int32),
                ("delta_window", C.c_int32)]


# name -> (restype, argtypes); every symbol include/lvsr_b200.h declares
_P = C.c_void_p
_I = C.c_int32
# lvsr_validate_fn(validate_user, utt, tokens, length); VALIDATE_FN() is the NULL callback
VALIDATE_FN = C.CFUNCTYPE(C.c_int32, _P, C.c_int32, C.POINTER(C.c_int64), C.c_int32)
SIGNATURES = {
    "lvsr_last_error": (C.c_char_p, []),
    "lvsr_version": (C.c_int, []),
    "lvsr_model_create": (C.c_int, [C.POINTER(LvsrConfig), C.POINTER(_P)]),
    "lvsr_model_create_bottom": (C.c_int, [C.POINTER(LvsrConfig), C.POINTER(LvsrBottomConfig), C.POINTER(_P)]),
    "lvsr_model_create_encoder": (C.c_int, [C.POINTER(LvsrConfig), C.POINTER(LvsrBottomConfig), C.c_int32, C.POINTER(_P)]),
    "lvsr_readout_max_width": (C.c_int, []),
    "lvsr_model_create_readout": (C.c_int, [C.POINTER(LvsrConfig), C.POINTER(LvsrBottomConfig), C.c_int32,
                                            C.POINTER(LvsrReadoutConfig), C.POINTER(_P)]),
    "lvsr_model_destroy": (C.c_int, [_P]),
    "lvsr_model_num_params": (C.c_int, [_P]),
    "lvsr_model_param_name": (C.c_char_p, [_P, C.c_int]),
    "lvsr_model_param_shape": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    "lvsr_model_set_param": (C.c_int, [_P, C.c_char_p, _P, C.c_int64]),
    "lvsr_model_get_param": (C.c_int, [_P, C.c_char_p, _P, C.c_int64]),
    "lvsr_model_flat_size": (C.c_int64, [_P]),
    "lvsr_model_param_offset": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "lvsr_model_flat_params": (C.c_void_p, [_P]),
    "lvsr_model_finalize": (C.c_int, [_P]),
    "lvsr_model_status": (C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "lvsr_model_decoder_plan": (C.c_int, [_P, C.POINTER(C.c_int32)]),
    "lvsr_model_encoder_plan": (C.c_int, [_P, _I, C.POINTER(C.c_int32)]),
    "lvsr_model_encoder_overlap": (C.c_int, [_P, _I, C.POINTER(C.c_int32)]),
    "lvsr_model_encoder_overlap_claims": (C.c_int, [_P, _I, C.POINTER(C.c_int32), C.c_int64]),
    "lvsr_encoded_length": (C.c_int, [_P, _I]),
    "lvsr_encoded_dim": (C.c_int, [_P]),
    "lvsr_encoder_forward": (C.c_int, [_P, _P, _P, _I, _I, _P, _P, _P]),
    "lvsr_preprocess": (C.c_int, [_P, _P, _I, _I, _P, _P]),
    "lvsr_cost_matrix": (C.c_int, [_P, _P, _P, _I, _I, _P, _P, _I, _P, _P, _P, _P, _P, _P]),
    "lvsr_model_set_criterion": (C.c_int, [_P, C.POINTER(LvsrCriterion)]),
    "lvsr_cost_matrix_groundtruth": (C.c_int, [_P, _P, _P, _I, _I, _P, _P, _I, _P, _I, _P, _P, _P, _P, _P, _P]),
    "lvsr_tle_matrices": (C.c_int, [_P, _P, _I, _P, _I, _I, _P, _P, _P]),
    "lvsr_initial_states": (C.c_int, [_P, _I, _I, _P, _P, _P, _P, _P, _P, _P]),
    "lvsr_logprobs": (C.c_int, [_P, _P, _P, _P, _I, _I, _P, _I, _P, _P, _P, _P, _P]),
    "lvsr_logprobs_lm": (C.c_int, [_P, _P, _P, _P, _I, _I, _P, _I, _P, _P, _P, _P, _P, _P]),
    "lvsr_next_states": (C.c_int, [_P, _P, _P, _P, _I, _I, _P, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "lvsr_beam_search_many": (C.c_int, [_P, _P, _P, _P, _I, _I, _P, _P, _I, _I, _I, C.c_double, C.c_double, _I, VALIDATE_FN,
                                        _P, C.POINTER(_P), _P]),
    "lvsr_search_result_count": (C.c_int, [_P, _I]),
    "lvsr_search_result_length": (C.c_int, [_P, _I, _I]),
    "lvsr_search_result_get": (C.c_int, [_P, _I, _I, _P, _P]),
    "lvsr_search_result_destroy": (C.c_int, [_P]),
    "lvsr_model_set_lm": (C.c_int, [_P, _I, _I, _P, C.c_int64, _P, _P, _P, C.POINTER(LvsrLmFusion)]),
    "lvsr_model_clear_lm": (C.c_int, [_P]),
    "lvsr_lm_initial_states": (C.c_int, [_P, _I, _P, _P, _P, _P]),
    "lvsr_lm_next_states": (C.c_int, [_P, _I, _P, _P, _P, _P, _P, _P, _P]),
    "lvsr_recognizer_cost_host": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P]),
    "lvsr_train_cost_and_grads": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, C.c_float, _P, _P, _P]),
    "lvsr_train_cost_and_grads_greedy": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, C.c_float, _P, _P, _P, _P, _P]),
    "lvsr_train_apply_updates": (C.c_int, [_P, _P, C.c_float, C.POINTER(LvsrTrainConfig), _P]),
    "lvsr_train_gradient_norm": (C.c_int, [_P, C.POINTER(C.c_float)]),
    "lvsr_train_reset": (C.c_int, [_P]),
    "lvsr_train_set_adaptive_clipping": (C.c_int, [_P, C.POINTER(LvsrAdaptiveClipping)]),
    "lvsr_train_clipping_threshold": (C.c_int, [_P, C.POINTER(C.c_double)]),
    "lvsr_alignment_stats": (C.c_int, [_P, _P, _P, _I, _I, _I, _P, _P]),
    "lvsr_train_set_adaptive_noise": (C.c_int, [_P, C.POINTER(LvsrAdaptiveNoise)]),
    "lvsr_train_get_noise_param": (C.c_int, [_P, C.c_int, _P, C.c_int64]),
    "lvsr_train_set_noise_param": (C.c_int, [_P, C.c_int, _P, C.c_int64]),
    "lvsr_train_noise_stats": (C.c_int, [_P, C.POINTER(C.c_double)]),
    "lvsr_train_noise_sample": (C.c_int, [_P, C.c_int64, _P, _P]),
    "lvsr_train_noise_params": (C.c_int, [_P, _P, _P]),
    "lvsr_train_noise_gradients": (C.c_int, [_P, _P, C.c_float, _P, _P]),
    "lvsr_train_set_regularization": (C.c_int, [_P, C.POINTER(LvsrRegularization)]),
    "lvsr_train_set_utterance_offset": (C.c_int, [_P, C.c_int64]),
    "lvsr_train_dropout_mask": (C.c_int, [_P, C.c_int64, C.c_int64, _I, _I, _I, _P, _P]),
    "lvsr_train_weight_noise_sample": (C.c_int, [_P, C.c_int64, _P, _P]),
    "lvsr_train_penalty_sum": (C.c_int, [_P, _P, _P]),
    "lvsr_frontend_create": (C.c_int, [C.POINTER(LvsrFbankOptions), C.POINTER(_P)]),
    "lvsr_frontend_destroy": (C.c_int, [_P]),
    "lvsr_frontend_num_frames": (C.c_int64, [_P, C.c_int64]),
    "lvsr_frontend_feature_dim": (C.c_int, [_P]),
    "lvsr_frontend_compute": (C.c_int, [_P, _P, C.c_int64, C.POINTER(C.c_int64), _I, _I, _P, _P, _P, _P]),
    "lvsr_frontend_accumulate_cmvn": (C.c_int, [_P, _P, _P, _I, _I, _P, _P]),
    "lvsr_frontend_apply_cmvn": (C.c_int, [_P, _P, _P, _I, _I, _P, _P]),
    "lvsr_frontend_dither_sample": (C.c_int, [_P, _I, _I, _P, _P]),
    "lvsr_launch_count": (C.c_int64, [C.c_int]),
    "lvsr_device_bytes": (C.c_int64, []),
    "lvsr_profile_enable": (C.c_int, [C.c_int]),
    "lvsr_profile_read": (C.c_int, [C.c_char_p, C.POINTER(C.c_double), C.POINTER(C.c_int64)]),
}

_lib = None


def load():
    """Load the shared library (once) and declare every signature."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "%s is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(attention-lvcsr_b200 has no CPU or PyTorch fallback)" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        msg = load().lvsr_last_error()
        raise RuntimeError("lvsr_b200: " + (msg.decode("utf-8", "replace") if msg else "error %d" % rc))
