"""CPU-only checks: oracle self-consistency, host logic, and that the C-ABI library loads
and exports every symbol include/lvsr_b200.h declares (no compute calls without a GPU)."""
import os
import re

import numpy as np
import pytest

from helpers import O, PYRAMID, ROOT, package


def _peaky(cfg, seed):
    params = O.init_params(cfg, seed=seed, scale=10.0)
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.W"] *= 40
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.b"][cfg["eos_label"]] = 24.0
    return params


def test_oracle_beam_costs_equal_cost_matrix_of_returned_sequences():
    """The invariant libs/blocks/tests/test_search.py:72-117 checks."""
    cfg = O.make_config(max_decoded_length_scale=2.0, **PYRAMID)
    params = _peaky(cfg, 17)
    rng = np.random.RandomState(0)
    x = rng.normal(size=(48, cfg["num_features"]))
    outs, costs = O.beam_search(cfg, params, x, 4)
    assert outs and all(o[-1] == cfg["eos_label"] for o in outs)
    assert costs == sorted(costs)
    for out, cost in zip(outs, costs):
        c, w, e = O.analyze(cfg, params, x, np.asarray(out))
        assert np.allclose(c.sum(), cost, rtol=1e-9)
        assert np.allclose(w.sum(axis=1), 1.0)


def test_oracle_greedy_equals_beam_one_prefix():
    cfg = O.make_config(max_decoded_length_scale=2.0, **PYRAMID)
    params = _peaky(cfg, 17)
    rng = np.random.RandomState(1)
    x = rng.normal(size=(56, cfg["num_features"]))
    att, m = O.context_computer(cfg, params, x[:, None, :])
    ys, _, _ = O.generate_greedy(cfg, params, att, m, 28)
    outs, _ = O.beam_search(cfg, params, x, 1)
    n = len(outs[0])
    assert list(ys[:n, 0]) == outs[0]


def test_oracle_window_priors_reduce_to_full_attention_when_wide():
    base = O.make_config(**PYRAMID)
    wide = O.make_config(prior=dict(type="window_around_median", before=1000, after=1000), **PYRAMID)
    params = O.init_params(base, seed=2, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(base, B=3, T=40, seed=3)
    a = O.recognizer_cost(base, params, x, m, labels, lm)
    b = O.recognizer_cost(wide, params, x, m, labels, lm)
    assert np.allclose(a, b, rtol=1e-12)


def test_oracle_float32_twin_close_to_float64():
    cfg = O.make_config(**PYRAMID)
    p64 = O.init_params(cfg, seed=4, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=2, T=40, seed=5)
    c64 = O.recognizer_cost(cfg, p64, x, m, labels, lm)
    c32 = O.recognizer_cost(cfg, O.cast_params(p64, np.float32), x.astype(np.float32), m.astype(np.float32),
                            labels, lm.astype(np.float32))
    assert c32.dtype == np.float32
    assert np.abs(c32 - c64).max() < 1e-3


def test_encoder_subsampling_shapes():
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=1)
    x, m, _, _ = O.synthetic_batch(cfg, B=2, T=41, seed=1)
    att, am = O.encoder(cfg, params, x, m)
    assert att.shape == (11, 2, 256) and am.shape == (11, 2)      # ceil(ceil(41/2)/2)
    assert np.array_equal(am, m[::4])


def test_library_exports_every_declared_symbol():
    pkg = package()
    header = open(os.path.join(ROOT, "include", "lvsr_b200.h")).read()
    declared = set(re.findall(r"\b(lvsr_[a-z_0-9]+)\s*\(", header))
    assert declared == set(pkg._lib.SIGNATURES), declared ^ set(pkg._lib.SIGNATURES)
    if not os.path.exists(pkg._lib.LIB_PATH):
        pytest.skip("liblvsr_b200.so not built in this checkout (run __graft_entry__.build())")
    lib = pkg._lib.load()
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.lvsr_version() >= 100


def test_config_struct_layout_matches_header():
    pkg = package()
    header = open(os.path.join(ROOT, "include", "lvsr_b200.h")).read()
    body = header[header.index("typedef struct {"):header.index("} lvsr_config;")]
    names = re.findall(r"\b(?:int32_t|double)\s+([^;]+);", body)
    fields = []
    for n in names:
        for part in n.split(","):
            fields.append(part.strip().split("[")[0])
    assert fields == [f[0] for f in pkg._lib.LvsrConfig._fields_]


def test_product_path_never_imports_the_oracle():
    pkg_dir = os.path.join(ROOT, "attention-lvcsr_b200")
    for dirpath, _, files in os.walk(pkg_dir):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in text and "from oracle" not in text, f


def test_smallest_and_unsupported_options():
    pkg = package()
    (rows, cols), vals = pkg.BeamSearch._smallest(np.array([[3, 6, 4], [1, 2, 7]]), 2)
    assert list(rows) == [1, 1] and list(cols) == [0, 1] and list(vals) == [1, 2]
    with pytest.raises(NotImplementedError):
        pkg.SpeechRecognizer(input_dims={"recordings": 40}, input_num_chars={}, eos_label=1, num_phonemes=4,
                             dim_dec=8, dims_bidir=[8], attention_type="content", conv_n=1)
    with pytest.raises(NotImplementedError):
        pkg.SpeechRecognizer(input_dims={"recordings": 40}, input_num_chars={}, eos_label=1, num_phonemes=4,
                             dim_dec=8, dims_bidir=[8], conv_n=1, post_merge_dims=[8], lm={"path": "x"})


def test_no_gpu_means_loud_failure():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    pkg = package()
    rec = pkg.SpeechRecognizer(input_dims={"recordings": 40}, input_num_chars={}, eos_label=31, num_phonemes=32,
                               dim_dec=128, dims_bidir=[128], conv_n=4, conv_num_filters=2, post_merge_dims=[128],
                               post_merge_activation=pkg.Maxout(2))
    with pytest.raises(RuntimeError):
        rec.encode(np.zeros((4, 1, 40), dtype=np.float32))


def test_step_rule_chains_map_onto_the_train_config():
    """algorithms._to_train_config accepts exactly the CompositeRule shapes lvsr/main.py:480-516 can build (in that
    order) and refuses anything else instead of approximating it."""
    A = package().algorithms
    wsj = dict(gradient_threshold=10.0, rules=["momentum", "adadelta"], scale=1.0, momentum=0.0, decay_rate=0.95,
               epsilon=1e-8, burn_in_steps=3)
    rule = A.step_rule_from_config(wsj, dict(max_norm=1.0))
    assert [type(c).__name__ for c in rule.components] == ["StepClipping", "Momentum", "AdaDelta", "Restrict",
                                                           "RemoveNotFinite", "BurnIn"]
    tc = A._to_train_config(rule, decay=0.01)
    assert (tc.gradient_threshold, tc.use_momentum, tc.scale, tc.momentum) == (10.0, 1, 1.0, 0.0)
    assert tc.use_adadelta == 1 and abs(tc.decay_rate - 0.95) < 1e-7 and abs(tc.epsilon - 1e-8) < 1e-15
    assert (tc.max_norm, tc.burn_in_steps) == (1.0, 3) and abs(tc.decay - 0.01) < 1e-9
    proto = A.step_rule_from_config(dict(gradient_threshold=100.0, scale=0.01, momentum=0.0))     # prototype_speech.yaml
    tc = A._to_train_config(proto)
    assert (tc.use_momentum, tc.use_adadelta, tc.max_norm, tc.burn_in_steps) == (1, 0, 0.0, 0)
    with pytest.raises(NotImplementedError):                # AdaDelta before Momentum: not a chain of lvsr/main.py
        A._to_train_config(A.CompositeRule([A.AdaDelta(), A.Momentum(0.1, 0.0), A.RemoveNotFinite(0.0)]))
    with pytest.raises(NotImplementedError):                # RemoveNotFinite with another scaler
        A._to_train_config(A.CompositeRule([A.Momentum(0.1, 0.0), A.RemoveNotFinite(1)]))
    with pytest.raises(NotImplementedError):                # max-norm over another axis
        A._to_train_config(A.CompositeRule([A.Restrict(A.VariableClipping(1.0, axis=1), "WEIGHT"), A.RemoveNotFinite(0.0)]))
    with pytest.raises(NotImplementedError):                # max-norm subjects without the lookup table (lvsr/main.py:494-496)
        A.step_rule_from_config(wsj, dict(max_norm=1.0, max_norm_exclude_lookup=True))
    assert len(A.step_rule_from_config(wsj, dict(max_norm=0.0, max_norm_exclude_lookup=True)).components) == 5
    with pytest.raises(ValueError):
        A.AdaDelta(decay_rate=2.0)                           # B/algorithms/__init__.py:481-482
    with pytest.raises(ValueError):
        A.GradientDescent(step_rule=rule)                    # no recognizer: nothing to differentiate
