"""attention-lvcsr_b200 -- H100-native hot path of rizar/attention-lvcsr.

The directory name contains a hyphen (it is the contract's name); import it through
``__graft_entry__.load_package()`` which registers it as ``attention_lvcsr_b200``.

Only what the path needs lives here: ``csrc/`` (sm_90a kernels + the C ABI of
include/lvsr_b200.h) and the host-side mirror of the reference's operator surface
(``SpeechRecognizer``, ``BeamSearch``, initialisation/config tokens), and the filterbank front end that
computes the recognizer's input from waveforms (``Fbank``, ``GlobalCmvn``).
"""
from . import _lib  # noqa: F401
from .bricks import (Constant, GatedRecurrent, Identity, IsotropicGaussian, Maxout,  # noqa: F401
                     Orthogonal, Rectifier, Tanh, Uniform)
from . import algorithms  # noqa: F401
from .algorithms import (AdaDelta, BurnIn, CompositeRule, GradientDescent, Momentum, RemoveNotFinite,  # noqa: F401
                         Restrict, Scale, StepClipping, VariableClipping, adaptive_clipping, clipping_rule,
                         step_rule_from_config)
from .frontend import Fbank, FbankOptions, GlobalCmvn  # noqa: F401
from .recognizer import SpeechRecognizer  # noqa: F401
from .search import BeamSearch, CandidateNotFoundError  # noqa: F401

__all__ = ["GradientDescent", "CompositeRule", "StepClipping", "Momentum", "AdaDelta", "VariableClipping", "Restrict",
           "RemoveNotFinite", "BurnIn", "Scale", "adaptive_clipping", "clipping_rule", "step_rule_from_config", "SpeechRecognizer", "BeamSearch", "CandidateNotFoundError", "Maxout", "Rectifier", "Tanh",
           "Identity", "GatedRecurrent", "IsotropicGaussian", "Constant", "Orthogonal", "Uniform", "Fbank", "FbankOptions",
           "GlobalCmvn"]
