"""Content-only attention (attention_type: content, the TIMIT baseline of the reference) on the GPU against the
float64 oracle: forward parity of every output, the persistent decoder against the step-wise kernels, the
equivalence with a zero-handler content_and_conv model, beam search, greedy generation, gradients and optimizer
steps, checkpoints and the compat entry points."""
import os
from collections import OrderedDict

import numpy as np
import pytest

import content_oracle as CO
from helpers import O, PYRAMID, SMALL, WSJ, package, rel_err

pytestmark = pytest.mark.gpu

def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _cfg(arch, **kw):
    return CO.make_config(**dict(arch, **kw))


def _make(cfg, params=None, attention_type="content"):
    pkg = package()
    act = {"maxout": pkg.Maxout(cfg["maxout_pieces"]), "relu": pkg.Rectifier()}[cfg["post_merge_activation"]]
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": cfg["num_features"]}, input_num_chars={}, eos_label=cfg["eos_label"],
        num_phonemes=cfg["num_phonemes"], dim_dec=cfg["dim_dec"], dims_bidir=cfg["dims_bidir"],
        subsample=cfg["subsample"], dim_matcher=cfg["dim_matcher"], post_merge_dims=cfg["post_merge_dims"],
        post_merge_activation=act, attention_type=attention_type,
        conv_n=cfg["conv_n"] if attention_type != "content" else None, conv_num_filters=cfg["conv_num_filters"],
        max_decoded_length_scale=cfg["max_decoded_length_scale"],
        enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent, data_prepend_eos=False)
    if params is not None:
        rec.set_parameter_values(params)
    return rec


class _env(object):
    def __init__(self, **kv):
        self.kv = kv

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.kv}
        os.environ.update(self.kv)

    def __exit__(self, *a):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _forward(rec, x, m, labels, lm):
    torch = _torch()
    att, attm = rec.encode(x, m)
    r = rec.cost_matrix(labels, lm, att, attm, return_all=True)
    torch.cuda.synchronize()
    return att.cpu().numpy(), {k: v.cpu().numpy() for k, v in r.items()}


def test_content_model_has_the_cont_att_parameter_table_at_abi_104():
    _torch()
    cfg = _cfg(SMALL)
    rec = _make(cfg)
    assert list(rec.parameter_shapes().items()) == list(CO.param_shapes(cfg).items())
    assert rec.generator.transition.attention.name == "cont_att"
    assert package()._lib.load().lvsr_version() == 104


@pytest.mark.parametrize("arch,B,T", [("SMALL", 16, 60), ("PYRAMID", 37, 80), ("WSJ", 64, 48)])
def test_content_forward_matches_oracle(arch, B, T):
    _torch()
    cfg = _cfg({"SMALL": SMALL, "PYRAMID": PYRAMID, "WSJ": WSJ}[arch])
    params = CO.init_params(cfg, seed=3, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=B, T=T, seed=B)
    rec = _make(cfg, params)
    with _env(LVSR_DEC_CHECK="1"):
        att, got = _forward(rec, x, m, labels, lm)
    assert rec.launch_status() == (0, 0)
    assert rec.decoder_plan()["kernel"] == "dec_content"
    want_att, want_attm = O.encoder(cfg, params, x, m)
    want = CO.cost_matrix(cfg, params, want_att, want_attm, labels, lm, return_all=True)
    assert rel_err(att, want_att) < 1e-4
    for k in ("costs", "weights", "states", "weighted_averages"):
        assert rel_err(got[k], want[k]) < 1e-4, (k, rel_err(got[k], want[k]))
    assert not got["energies"].any()
    # the step-wise kernels compute the same thing as the persistent decoder
    with _env(LVSR_NO_DEC_SCAN="1"):
        _, step = _forward(rec, x, m, labels, lm)
    for k in ("costs", "weights", "states", "weighted_averages"):
        assert rel_err(step[k], got[k]) < 1e-5, (k, rel_err(step[k], got[k]))
    assert not step["energies"].any()
    assert rel_err(rec.cost(x, m, labels, lm), got["costs"]) < 1e-6


def test_content_forward_at_a_long_timit_like_length():
    """T' = 2000 encoded frames (TIMIT: three unsubsampled layers) on the persistent decoder."""
    _torch()
    cfg = _cfg(dict(num_features=40, dims_bidir=[128], subsample=[1], dim_dec=128, dim_matcher=128, num_phonemes=63,
                    post_merge_dims=[128], maxout_pieces=2))
    params = CO.init_params(cfg, seed=5, scale=10.0)
    x, m, labels, lm = O.synthetic_batch(cfg, B=4, T=2000, seed=2, label_div=100)
    rec = _make(cfg, params)
    with _env(LVSR_DEC_CHECK="1"):
        att, got = _forward(rec, x, m, labels, lm)
    assert rec.decoder_plan()["kernel"] == "dec_content"
    want_att, want_attm = O.encoder(cfg, params, x, m)
    want = CO.cost_matrix(cfg, params, want_att, want_attm, labels, lm, return_all=True)
    for k in ("costs", "weights", "states", "weighted_averages"):
        assert rel_err(got[k], want[k]) < 1e-4, (k, rel_err(got[k], want[k]))
    assert not got["energies"].any()


def test_content_equals_conv_model_with_zero_handler():
    _torch()
    cfg = _cfg(PYRAMID)
    params = CO.init_params(cfg, seed=4, scale=10.0)
    ccfg = O.make_config(**PYRAMID)
    cparams = OrderedDict((k.replace("cont_att", "conv_att"), v) for k, v in params.items())     # same order of names
    cparams[O._ATT + "/handler.W"] = np.zeros((ccfg["conv_num_filters"], ccfg["dim_matcher"]))
    cparams[O._ATT + "/conv1d.filters"] = np.random.RandomState(0).normal(size=(ccfg["conv_num_filters"], 2 * ccfg["conv_n"] + 1))
    x, m, labels, lm = O.synthetic_batch(cfg, B=16, T=64, seed=9)
    _, a = _forward(_make(cfg, params), x, m, labels, lm)
    _, b = _forward(_make(ccfg, cparams, "content_and_conv"), x, m, labels, lm)
    assert rel_err(a["costs"], b["costs"]) < 2e-6
    assert np.abs(a["weights"] - b["weights"]).max() < 2e-6


def test_content_initial_states_are_zero_weights():
    torch = _torch()
    rec = _make(_cfg(SMALL), CO.init_params(_cfg(SMALL), seed=1))
    st = rec._initial_states(17, 3)
    torch.cuda.synchronize()
    assert not st["weights"].any() and not st["energies"].any()


@pytest.mark.parametrize("beam_size,stop_on,char_discount", [(1, "patience", 0), (10, "patience", 0.0),
                                                             (10, "optimistic_future_cost", 0.1)])
def test_content_beam_search_many_equals_oracle(beam_size, stop_on, char_discount):
    _torch()
    cfg = _cfg(PYRAMID, max_decoded_length_scale=3.0)
    params = CO.init_params(cfg, seed=11, scale=10.0)
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.W"] *= 10.0
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.b"][cfg["eos_label"]] = 1.0
    rng = np.random.RandomState(5)
    utts = [rng.normal(size=(T, cfg["num_features"])) for T in (64, 37, 52, 64, 45, 30)]
    rec = _make(cfg, params)
    rec.init_beam_search(beam_size)
    got = rec.beam_search_many([{"recordings": u} for u in utts], stop_on=stop_on, char_discount=char_discount,
                               raise_on_failure=False)
    n_found = 0
    for u, g in zip(utts, got):
        try:
            want = CO.beam_search(cfg, params, u, beam_size, stop_on=stop_on, char_discount=char_discount)
        except O.CandidateNotFoundError:
            assert g is None
            continue
        n_found += 1
        assert g is not None and g[0] == want[0]
        assert np.allclose(g[1], want[1], rtol=1e-3, atol=5e-3)
    assert n_found >= 1


def test_content_greedy_generate_equals_oracle():
    _torch()
    cfg = _cfg(SMALL)
    params = CO.init_params(cfg, seed=3, scale=10.0)
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.W"] *= 8.0
    rec = _make(cfg, params)
    x, m, _, _ = O.synthetic_batch(cfg, B=3, T=40, seed=7)
    att, attm = O.encoder(cfg, params, x, m)
    ys, costs, _ = CO.generate_greedy(cfg, params, att, attm, 6)
    g = rec.generate(x, m, n_steps=6, sample=False)
    assert np.array_equal(g["outputs"], ys)
    assert rel_err(g["costs"], costs) < 1e-3
    assert rec.sample({"recordings": x[:, 0]}, n_steps=4).shape == (4, 1)


@pytest.mark.parametrize("arch,B,T", [("PYRAMID", 18, 40), ("WSJ", 8, 48)])
def test_content_gradients_match_oracle(arch, B, T):
    _torch()
    pkg = package()
    cfg = _cfg({"PYRAMID": PYRAMID, "WSJ": WSJ}[arch])
    params = CO.init_params(cfg, seed=7, scale=10.0)
    batch = O.synthetic_batch(cfg, B=B, T=T, seed=12)
    rec = _make(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
    cost, grads = algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
    want_cost, want = CO.cost_and_grads(cfg, params, *batch)
    assert set(grads) == set(want)
    assert abs(cost - want_cost) <= 1e-4 * abs(want_cost)
    for k, w in want.items():
        assert np.abs(grads[k] - w).max() <= 1e-4 * np.abs(w).max() + 1e-9, (k, rel_err(grads[k], w))


def test_content_two_optimizer_steps_equal_oracle():
    _torch()
    from oracle import lvsr_oracle_grad as G
    pkg = package()
    cfg = _cfg(PYRAMID)
    params = CO.init_params(cfg, seed=5, scale=10.0)
    tc = G.make_train_config(gradient_threshold=2.0, rules=("momentum", "adadelta"), scale=0.05, momentum=0.5,
                             decay_rate=0.95, epsilon=1e-6, max_norm=1.0)
    rec = _make(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(tc, dict(max_norm=1.0)))
    algo.initialize()
    ref, state = OrderedDict((k, v.copy()) for k, v in params.items()), {}
    for step in range(2):
        batch = O.synthetic_batch(cfg, B=4, T=40, seed=100 + step)
        ref, ref_cost, _ = CO.train_step(cfg, ref, state, batch, tc)
        algo.process_batch(dict(zip(algo.SOURCES, batch)))
        assert abs(float(algo.last_cost.item()) - ref_cost) <= 1e-4 * abs(ref_cost)
        got = rec.get_parameter_values()
        for k, v in ref.items():
            assert np.abs(got[k] - v).max() <= 2e-5 * max(1.0, np.abs(v).max()) + 1e-6, (step, k)


def test_content_checkpoint_round_trip_and_conv_checkpoint(tmp_path, caplog):
    _torch()
    cfg = _cfg(SMALL)
    params = CO.init_params(cfg, seed=3, scale=10.0)
    rec = _make(cfg, params)
    path = str(tmp_path / "model.tar")
    rec.save_params(path)
    rec2 = _make(cfg)
    assert rec2.load_params(path) == dict(unknown=[], missing=[])
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=20, seed=1)
    assert np.array_equal(rec.cost(x, m, labels, lm), rec2.cost(x, m, labels, lm))
    ccfg = O.make_config(**SMALL)
    conv = _make(ccfg, O.init_params(ccfg, seed=3), "content_and_conv")
    cpath = str(tmp_path / "conv.tar")
    conv.save_params(cpath)
    with caplog.at_level("ERROR"):
        info = _make(cfg).load_params(cpath)
    assert sorted(info["unknown"]) == sorted(k for k in O.param_shapes(ccfg) if "conv_att" in k)
    assert sorted(info["missing"]) == sorted(k for k in CO.param_shapes(cfg) if "cont_att" in k)
    assert "unknown parameter names" in caplog.text and "missing values for parameters" in caplog.text


def test_content_compat_entry_points(tmp_path, capsys):
    _torch()
    import sys
    import tarfile
    import compat_helpers as CH
    if CH.COMPAT not in sys.path:
        sys.path.insert(0, CH.COMPAT)
    import lvsr.config as C
    import lvsr.main as M
    exp = CH.write_experiment(tmp_path)
    base = open(exp["base"]).read().replace("attention_type: content_and_conv\n    conv_n: 8\n    conv_num_filters: 4\n",
                                             "attention_type: content\n")
    assert "attention_type: content\n" in base
    open(exp["base"], "w").write(base)
    cfg = C.Configuration(exp["child"], None, [])
    cfg["cmd_args"] = {}
    save = str(tmp_path / "run")
    M.train_multistage(cfg, save, "", None, "")
    with tarfile.open(os.path.join(save, "main.tar")) as tar:
        names = np.load(__import__("io").BytesIO(tar.extractfile("_parameters").read())).files
    assert any("cont_att" in n for n in names) and not any("conv_att" in n for n in names)
    capsys.readouterr()
    single = C.Configuration(exp["base"], None, [("monitoring.search.beam_size", "2")])
    decoded = str(tmp_path / "decoded.txt")
    M.search(single, None, os.path.join(save, "main.tar"), "valid", None, None, decoded, False, 1)
    assert "Average CER:" in capsys.readouterr().out
    M.sample(single, None, os.path.join(save, "main.tar"), "valid")
    assert "Utterance 2" in capsys.readouterr().out
