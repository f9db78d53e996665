"""The deep readout (net.post_merge_dims of 2 to 4 entries) on the GPU against the float64 oracle
(tests/readout_oracle.py): teacher-forced costs on both decoder plans, the state functions, greedy generation and
sampling, beam search, gradients and optimizer steps, checkpoints and pickling, and a depth-1 model made through the
new entry point against one made through lvsr_model_create_encoder.

The decoder's recurrence and the encoder do not read the readout, so the oracle's costs are computed from the
encoder output the GPU produced (rounded to float32), through the oracle's decoder of the model's attention type and
decoder depth: what is compared is the readout's part, at every depth, activation, width and vocabulary."""
import ctypes
import pickle
from collections import OrderedDict

import numpy as np
import pytest

import content_oracle as CO
import readout_oracle as RO
import stack_oracle as SO
from helpers import O, f32, make_recognizer, package, rel_err
from oracle import lvsr_oracle_grad as G

pytestmark = pytest.mark.gpu

MLP = RO.PM + "/mlp/"


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _cfg(dims, act="relu", V=32, attention="content_and_conv", stack=False, use_states=True, **kw):
    base = dict(num_features=40, dims_bidir=[128], subsample=[1], dim_dec=128, dim_matcher=128, conv_n=8,
                conv_num_filters=4, num_phonemes=V, post_merge_dims=dims[:1], post_merge_activation=act,
                maxout_pieces=1, use_states_for_readout=use_states, max_decoded_length_scale=2.0)
    base.update(kw)
    if stack:
        cfg = SO.make_config(attention_type=attention, **base)
    elif attention == "content":
        cfg = CO.make_config(**base)
    else:
        cfg = O.make_config(**base)
    cfg["post_merge_dims"] = [int(d) for d in dims]
    return cfg


def _params(cfg, seed=3, gain=10.0):
    """The model's oracle parameters with the deep MLP: weights large enough that every layer matters."""
    mod = SO if cfg.get("dec_stack") == 2 else (CO if cfg.get("attention_type") == "content" else O)
    base = mod.init_params(dict(cfg, post_merge_dims=cfg["post_merge_dims"][:1]), seed=seed, scale=gain)
    rng = np.random.RandomState(seed + 100)
    dims, V = cfg["post_merge_dims"], cfg["num_phonemes"]
    out = OrderedDict()
    for k, v in base.items():            # in the table's order: the MLP's Linears follow post_merge/bias.b
        if k.startswith(MLP):
            continue
        out[k] = v
        if k == RO.PM + "/bias.b":
            for j in range(len(dims)):
                din, dout = dims[j], dims[j + 1] if j + 1 < len(dims) else V
                out[RO.linear_name(j) + ".b"] = rng.normal(0, 0.3, size=(dout,))
                out[RO.linear_name(j) + ".W"] = rng.normal(0, 1.5 / np.sqrt(din), size=(din, dout))
    return out


def _oracle_costs(cfg, params, att, attm, labels, lmask):
    """Teacher-forced costs and alignments of the deep model from the attended sequence."""
    shallow = RO.shallow_params(cfg, params)
    if cfg.get("dec_stack") == 2:
        r = SO.cost_matrix(cfg, shallow, att, attm, labels, lmask, return_all=True)
        wide = SO.wide_params(cfg, params)
    else:
        r = (CO if cfg.get("attention_type") == "content" else O).cost_matrix(cfg, shallow, att, attm, labels, lmask,
                                                                               return_all=True)
        wide = params
    logits = RO.readout(cfg, wide, r["states"], r["weighted_averages"])
    costs = -np.take_along_axis(O.log_softmax(logits), labels[..., None], axis=-1)[..., 0]
    if lmask is not None:
        costs = costs * lmask
    return costs, r["weights"], logits


def _encode(rec, x, m):
    att, attm = rec.encode(x, m)
    return att, attm, f32(att.cpu().numpy()), f32(attm.cpu().numpy())


CASES = [
    ([128, 128], "tanh", 32, "content_and_conv", False, True),
    ([128, 256, 72], "relu", 5, "content_and_conv", False, True),
    ([200, 8, 64, 512], "identity", 128, "content_and_conv", False, False),
    ([256, 200], "maxout", 32, "content", False, True),
    ([72, 512], "relu", 128, "content_and_conv", True, True),
    ([128, 1408], "tanh", 32, "content", True, False),
]


@pytest.mark.parametrize("dims,act,V,attention,stack,use_states", CASES)
@pytest.mark.parametrize("stepwise", [False, True])
def test_costs_and_analyze_match_oracle(dims, act, V, attention, stack, use_states, stepwise, monkeypatch):
    _torch()
    if stepwise:
        monkeypatch.setenv("LVSR_NO_DEC_SCAN", "1")
    cfg = _cfg(dims, act, V, attention, stack, use_states)
    params = _params(cfg)
    rec = make_recognizer(cfg, params)
    x, m, labels, lm = O.synthetic_batch(cfg, B=5, T=36, seed=11)
    att, attm, att64, attm64 = _encode(rec, x, m)
    got = rec.cost_matrix(labels, lm, att, attm).cpu().numpy()
    ran = rec.decoder_plan()["ran"]
    assert ran == (not stepwise and not stack)
    want, _, _ = _oracle_costs(cfg, params, att64, attm64, labels, lm)
    assert np.abs(got - want).max() <= 2e-4 * max(1.0, np.abs(want).max()), rel_err(got, want)
    # analyze: one utterance, prediction scored
    u = x[:, 0]
    costs, weights, _ = rec.analyze({"recordings": u}, labels[:, 0])
    a1, m1, a64, m64 = _encode(rec, u[:, None, :], np.ones((u.shape[0], 1), np.float32))
    w_costs, w_weights, _ = _oracle_costs(cfg, params, a64, m64, labels[:, :1], None)
    assert np.abs(costs - w_costs[:, 0]).max() <= 2e-4 * max(1.0, np.abs(w_costs).max())
    assert np.abs(weights - w_weights[:, 0]).max() <= 1e-3


@pytest.mark.parametrize("dims,act,V", [([128, 128], "tanh", 32), ([128, 64, 256], "relu", 5),
                                        ([256, 256, 256, 256], "identity", 128)])
def test_logprobs_greedy_and_sample(dims, act, V):
    _torch()
    cfg = _cfg(dims, act, V)
    params = _params(cfg, seed=5)
    rec = make_recognizer(cfg, params)
    x, m, _, _ = O.synthetic_batch(cfg, B=3, T=40, seed=7)
    att, attm, att64, attm64 = _encode(rec, x, m)
    ctx = dict(attended=att, attended_mask=attm, preprocessed=rec.preprocess(att))
    st = rec._initial_states(att.shape[0], 3)
    got = rec._logprobs(ctx, st).cpu().numpy()
    ost = RO.initial_states(cfg, params, 3, att64)
    want = RO.logprobs_computer(cfg, params, att64, attm64, ost)
    assert np.abs(got - want).max() <= 2e-4 * max(1.0, np.abs(want).max())
    ys, costs, _ = RO.generate_greedy(cfg, params, att64, attm64, 6)
    g = rec.generate(x, m, n_steps=6, sample=False)
    assert np.array_equal(g["outputs"], ys)
    assert rel_err(g["costs"], costs) < 1e-3
    # sampling: every emitted symbol is scored with the oracle's -log p along the sampled path
    s = rec.generate(x, m, n_steps=5, sample=True, seed=3)
    ost = RO.initial_states(cfg, params, 3, att64)
    for i in range(5):
        lp = RO.logprobs_computer(cfg, params, att64, attm64, ost)
        y = s["outputs"][i]
        assert np.abs(s["costs"][i] - lp[np.arange(3), y]).max() <= 2e-3 * max(1.0, np.abs(lp).max())
        ost = RO.next_state_computer(cfg, params, att64, attm64, ost, y)


@pytest.mark.parametrize("beam_size,stop_on", [(1, "patience"), (10, "patience"), (10, "optimistic_future_cost"),
                                               (200, "patience")])
def test_beam_search_many_matches_oracle(beam_size, stop_on):
    _torch()
    cfg = _cfg([128, 128, 64], "tanh", 32)
    params = _params(cfg, seed=9)
    params[RO.linear_name(2) + ".b"][cfg["eos_label"]] += 3.0
    rec = make_recognizer(cfg, params)
    rng = np.random.RandomState(5)
    utts = [rng.normal(size=(T, cfg["num_features"])) for T in (40, 27, 33)][:2 if beam_size == 200 else 3]
    rec.init_beam_search(beam_size)
    got = rec.beam_search_many([{"recordings": u} for u in utts], stop_on=stop_on, raise_on_failure=False)
    found = 0
    for u, g in zip(utts, got):
        try:
            want = RO.beam_search(cfg, params, u, beam_size, stop_on=stop_on)
        except O.CandidateNotFoundError:
            assert g is None
            continue
        found += 1
        assert g is not None and g[0] == want[0]
        assert np.allclose(g[1], want[1], rtol=1e-3, atol=5e-3)
    assert found >= 1


@pytest.mark.parametrize("dims,act", [([128, 128], "tanh"), ([128, 256, 64], "relu"), ([128, 72, 72, 8], "identity")])
def test_gradients_match_oracle(dims, act):
    _torch()
    pkg = package()
    cfg = _cfg(dims, act)
    params = _params(cfg, seed=7, gain=3.0)
    batch = O.synthetic_batch(cfg, B=4, T=30, seed=12)
    rec = make_recognizer(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
    cost, grads = algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
    want_cost, want = RO.cost_and_grads(cfg, params, *batch)
    assert set(grads) == set(want)
    assert abs(cost - want_cost) <= 1e-4 * abs(want_cost)
    gmax = max(np.abs(w).max() for w in want.values())
    for k, w in want.items():
        assert np.abs(grads[k] - w).max() <= 1e-4 * np.abs(w).max() + 1e-6 * gmax, (k, rel_err(grads[k], w))


def test_two_optimizer_steps_equal_oracle():
    _torch()
    pkg = package()
    cfg = _cfg([128, 128, 64], "tanh")
    params = _params(cfg, seed=5, gain=3.0)
    tc = G.make_train_config(gradient_threshold=2.0, rules=("momentum", "adadelta"), scale=0.05, momentum=0.5,
                             decay_rate=0.95, epsilon=1e-6, max_norm=1.0)
    rec = make_recognizer(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(tc, dict(max_norm=1.0)))
    algo.initialize()
    ref, state = OrderedDict((k, v.copy()) for k, v in params.items()), {}
    for step in range(2):
        batch = O.synthetic_batch(cfg, B=4, T=30, seed=100 + step)
        ref, ref_cost, _ = RO.train_step(cfg, ref, state, batch, tc)
        algo.process_batch(dict(zip(algo.SOURCES, batch)))
        assert abs(float(algo.last_cost.item()) - ref_cost) <= 1e-4 * abs(ref_cost)
        got = rec.get_parameter_values()
        for k, v in ref.items():
            assert np.abs(got[k] - v).max() <= 2e-5 * max(1.0, np.abs(v).max()) + 1e-6, (step, k)
    # max-norm treats every linear_j.W as a WEIGHT
    for j in range(3):
        W = rec.get_parameter_values()[RO.linear_name(j) + ".W"].astype(np.float64)
        assert (np.sqrt((W ** 2).sum(axis=0)) <= 1.0 + 1e-5).all()


def test_checkpoint_round_trip_and_pickle(tmp_path):
    _torch()
    cfg = _cfg([128, 256, 64], "relu")
    params = _params(cfg, seed=3)
    rec = make_recognizer(cfg, params)
    path = str(tmp_path / "model.tar")
    rec.save_params(path)
    import tarfile
    with tarfile.open(path) as tar:
        names = np.load(__import__("io").BytesIO(tar.extractfile("_parameters").read())).files
    assert "|recognizer|generator|readout|post_merge|mlp|linear_1.W" in names
    rec2 = make_recognizer(cfg)
    assert rec2.load_params(path) == dict(unknown=[], missing=[])
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=20, seed=1)
    want = rec.cost(x, m, labels, lm)
    assert np.array_equal(want, rec2.cost(x, m, labels, lm))
    rec3 = pickle.loads(pickle.dumps(rec))
    assert rec3.net["post_merge_dims"] == [128, 256, 64]
    assert np.array_equal(want, rec3.cost(x, m, labels, lm))


def test_depth_one_through_the_new_entry_is_bit_identical():
    """lvsr_model_create_readout with a one-layer readout is lvsr_model_create_encoder: same table, same launches, the
    same bits in costs, search results and gradients."""
    torch = _torch()
    pkg = package()
    lib = pkg._lib.load()
    cfg = O.make_config(num_features=40, dims_bidir=[128], subsample=[1], dim_dec=128, dim_matcher=256, conv_n=8,
                        conv_num_filters=4, num_phonemes=32, post_merge_dims=[128], maxout_pieces=2)
    params = O.init_params(cfg, seed=4, scale=10.0)
    old = make_recognizer(cfg, params)
    new = make_recognizer(cfg)
    c = new._make_config()
    ro = pkg._lib.LvsrReadoutConfig()
    ro.num_layers, ro.dims[0] = 1, 128
    h = ctypes.c_void_p()
    with torch.cuda.device(new.device):
        pkg._lib.check(lib.lvsr_model_create_readout(ctypes.byref(c), None, 1, ctypes.byref(ro), ctypes.byref(h)))
    new._handle = h
    new.set_parameter_values(params)
    assert old.parameter_shapes() == new.parameter_shapes()
    x, m, labels, lm = O.synthetic_batch(cfg, B=4, T=30, seed=2)
    counts, costs, searches, grads = [], [], [], []
    for rec in (old, new):
        torch.cuda.synchronize()
        lib.lvsr_launch_count(1)
        costs.append(rec.cost(x, m, labels, lm))
        counts.append(lib.lvsr_launch_count(1))
        rec.init_beam_search(10)
        searches.append(rec.beam_search({"recordings": x[:, 0]}))
        algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
        grads.append(algo.cost_and_gradients(dict(zip(algo.SOURCES, (x, m, labels, lm))))[1])
    assert counts[0] == counts[1]
    assert np.array_equal(costs[0], costs[1])
    assert searches[0][0] == searches[1][0] and np.array_equal(searches[0][1], searches[1][1])
    for k in grads[0]:
        assert np.array_equal(grads[0][k], grads[1][k]), k


def test_non_default_stream():
    torch = _torch()
    cfg = _cfg([128, 128], "tanh")
    params = _params(cfg)
    rec = make_recognizer(cfg, params)
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=24, seed=6)
    want = rec.cost(x, m, labels, lm)
    s = torch.cuda.Stream(device=rec.device)
    with torch.cuda.stream(s):
        att, attm = rec.encode(x, m)
        got = rec.cost_matrix(labels, lm, att, attm)
    s.synchronize()
    assert np.abs(got.cpu().numpy() - want).max() <= 1e-5 * max(1.0, np.abs(want).max())


def test_refused_readout_leaves_the_library_usable():
    _torch()
    pkg = package()
    lib = pkg._lib.load()
    cfg = _cfg([128, 128], "tanh")
    rec = make_recognizer(cfg, _params(cfg))
    c = rec._make_config()
    ro = pkg._lib.LvsrReadoutConfig()
    ro.num_layers, ro.dims[0], ro.dims[1] = 2, 128, 12
    h = ctypes.c_void_p()
    assert lib.lvsr_model_create_readout(ctypes.byref(c), None, 1, ctypes.byref(ro), ctypes.byref(h)) != 0
    assert "multiple of 8" in lib.lvsr_last_error().decode()
    x, m, labels, lm = O.synthetic_batch(cfg, B=2, T=20, seed=1)
    assert np.isfinite(rec.cost(x, m, labels, lm)).all()


# ---- the readout's other emitters, the forward-only encoder, the regularisers and compat ---------------------------


def _peaky_deep(seed=9):
    cfg = _cfg([128, 128, 64], "tanh", 32)
    params = _params(cfg, seed=seed)
    params[RO.linear_name(2) + ".b"][cfg["eos_label"]] += 3.0
    return cfg, params


def _search_both(rec, cfg, params, beam_size, computers, n=3):
    rng = np.random.RandomState(5)
    utts = [rng.normal(size=(T, cfg["num_features"])) for T in (40, 27, 33)][:n]
    rec.init_beam_search(beam_size)
    got = rec.beam_search_many([{"recordings": u} for u in utts], raise_on_failure=False)
    found = 0
    for u, g in zip(utts, got):
        try:
            want = O.beam_search(cfg, params, u, beam_size, computers=computers)
        except O.CandidateNotFoundError:
            assert g is None
            continue
        found += 1
        assert g is not None and g[0] == want[0]
        assert np.allclose(g[1], want[1], rtol=1e-3, atol=5e-3)
    assert found >= 1


@pytest.mark.parametrize("name", ["mse_gain", "mse_reward"])
def test_task_loss_cost_and_search(name):
    """RewardRegressionEmitter on the deep readout: the costs of the criterion over -logits, and its beam search."""
    _torch()
    import tle_oracle as TO
    cfg, params = _peaky_deep()
    rec = make_recognizer(cfg, params, criterion=dict(name=name, min_reward=-1.0))
    x, m, labels, lm = O.synthetic_batch(cfg, B=4, T=36, seed=13)
    att, attm, att64, attm64 = _encode(rec, x, m)
    got = rec.cost_matrix(labels, lm, att, attm).cpu().numpy()
    logits = RO.cost_matrix(cfg, params, att64, attm64, labels, lm, emitter="readouts")
    rewards, gains = TO.reward_op(labels, labels, cfg["num_phonemes"], cfg["eos_label"])
    want = TO.tle_cost(name, logits, labels, rewards, gains, -1.0, lm)
    assert np.abs(got - want).max() <= 2e-4 * max(1.0, np.abs(want).max()), rel_err(got, want)
    shallow = RO.shallow_params(cfg, params)
    comps = dict(initial=lambda a: TO.initial_states(cfg, shallow, 1, a),
                 logprobs=lambda a, mm, st: -RO.logits_computer(cfg, params, a, mm, st),
                 next=lambda a, mm, st, y: RO.next_state_computer(cfg, params, a, mm, st, y))
    _search_both(rec, cfg, params, 10, comps)


def test_language_model_fused_cost_and_search(tmp_path):
    """ShallowFusionReadout + LMEmitter on the deep readout's logits, in the teacher-forced costs and the search."""
    _torch()
    import lm_oracle as LO
    cfg, params = _peaky_deep()
    V = cfg["num_phonemes"]
    S, start, arcs = LO.char_ngram(V, seed=7, n_tri=60, dup=6, dead=2)
    path = str(tmp_path / "lm.fst")
    cmap = LO.to_file(path, V, S, start, arcs, seed=2)
    fst = LO.from_tables(package().lm.load(path, cmap, V))
    rec = make_recognizer(cfg, params, lm=dict(path=path, weight=0.5, no_transition_cost=20.0), character_map=cmap)
    o = rec.lm
    x, m, labels, lm = O.synthetic_batch(cfg, B=4, T=36, seed=13)
    att, attm, att64, attm64 = _encode(rec, x, m)
    got = rec.cost_matrix(labels, lm, att, attm).cpu().numpy()
    logits = RO.cost_matrix(cfg, params, att64, attm64, labels, lm, emitter="readouts")
    add = LO.lm_path(fst, labels, lm, V, o["no_transition_cost"])
    want = np.take_along_axis(LO.fused_costs(logits, add, o), labels[..., None], axis=-1)[..., 0] * lm
    assert np.allclose(got, want, rtol=1e-4, atol=1e-4), np.abs(got - want).max()
    comps = LO.computers(cfg, RO.shallow_params(cfg, params), fst, o)
    comps["logprobs"] = lambda a, mm, st: LO.fused_costs(RO.logits_computer(cfg, params, a, mm, st), st["lm_add"], o)
    _search_both(rec, cfg, params, 10, comps)


def test_forward_only_encoder():
    """A deep readout behind a forward-only encoder: costs on both decoder plans and the gradients of the readout."""
    _torch()
    pkg = package()
    import unidirectional_oracle as U
    cfg = _cfg([128, 96, 64], "relu", 32)
    rec = make_recognizer(cfg, None, bidir=False)
    values = rec.initial_values(rec.parameter_shapes(), seed=4)
    deep = _params(dict(cfg, dims_bidir=[64]), seed=4)         # the decoder of a 64-wide encoded sequence
    params = OrderedDict((k, deep.get(k, v)) for k, v in values.items())
    params = OrderedDict((k, np.asarray(v, np.float64) * (10.0 if "/encoder/" in k and k.endswith(".W") else 1.0))
                         for k, v in params.items())
    rec.set_parameter_values(params)
    x, m, labels, lm = O.synthetic_batch(cfg, B=4, T=32, seed=3)
    att, attm, att64, attm64 = _encode(rec, x, m)
    assert att.shape[2] == 128
    dcfg = U.decoder_config(dict(cfg, bidir=False))
    want, _, _ = _oracle_costs(dcfg, params, att64, attm64, labels, lm)
    for stepwise in (False, True):
        import os
        if stepwise:
            os.environ["LVSR_NO_DEC_SCAN"] = "1"
        try:
            got = rec.cost_matrix(labels, lm, att, attm).cpu().numpy()
        finally:
            os.environ.pop("LVSR_NO_DEC_SCAN", None)
        assert np.abs(got - want).max() <= 2e-4 * max(1.0, np.abs(want).max()), (stepwise, rel_err(got, want))
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
    _, grads = algo.cost_and_gradients(dict(zip(algo.SOURCES, (x, m, labels, lm))))
    # the readout's gradients from the tape of the GPU's encoder output: the torch mirror on the attended sequence
    import torch
    p = OrderedDict((k, torch.tensor(np.asarray(v, np.float64), requires_grad=True)) for k, v in params.items()
                    if k.startswith(O._GEN + "/readout/") or not k.startswith("/recognizer/encoder/"))
    costs = RO._cost_matrix_torch(dcfg, p, torch.as_tensor(att64), torch.as_tensor(attm64), labels, torch.as_tensor(lm))
    names = [k for k in p if k.startswith(RO.PM)]
    g = torch.autograd.grad(costs.sum() / labels.shape[1], [p[k] for k in names])
    for k, w in zip(names, g):
        w = w.numpy()
        assert np.abs(grads[k] - w).max() <= 1e-4 * np.abs(w).max() + 1e-9, (k, rel_err(grads[k], w))


@pytest.mark.parametrize("reg", ["dropout", "noise", "penalty"])
def test_regularised_gradients_match_the_oracle(reg, monkeypatch):
    """Dropout, weight noise and the alignment penalty over a deep readout: the cost and every gradient against the
    regularisation oracle on the replayed draws, with the deep readout's torch mirror as its cost matrix."""
    _torch()
    import regularization_oracle as REG
    import test_gpu_regularization as TR
    monkeypatch.setattr(G, "_cost_matrix", RO._cost_matrix_torch)
    # the regularisation tests' attention (M 256, 10 filters, weights x 10): with flatter alignments consecutive
    # cumulative alignments tie within rounding, and the penalty's max(., 0) takes a different side of its kink in
    # float32 than in float64, whatever the readout
    cfg = _cfg([128, 128, 64], "tanh", 32, dim_matcher=256, conv_num_filters=10)
    params = OrderedDict((k, f32(v)) for k, v in _params(cfg, seed=21, gain=10.0).items())
    setting = {"dropout": dict(dropout=True), "noise": dict(noise=TR.LEVEL), "penalty": dict(penalty_coof=TR.COOF)}[reg]
    batch = O.synthetic_batch(cfg, B=3, T=36, seed=22)
    algo = TR._algorithm(make_recognizer(cfg, params), dict(setting, seed=9))
    cost, grads = algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
    mult, eps = TR._draws(algo, cfg, setting, 0, batch)
    TR._check(cfg, params, batch, cost, grads, mult, eps, setting.get("penalty_coof", 0.0))
    _, clean = RO.cost_and_grads(cfg, params, *batch)
    assert any(np.abs(clean[k] - grads[k]).max() > 1e-2 * np.abs(clean[k]).max() for k in clean)
    assert REG is not None


def test_adaptive_noise_two_steps_match_the_oracle(monkeypatch):
    _torch()
    import adaptive_noise_oracle as AN
    import test_gpu_adaptive_noise as TA
    monkeypatch.setattr(G, "_cost_matrix", RO._cost_matrix_torch)
    cfg = _cfg([128, 128, 64], "tanh", 32)
    params = _params(cfg, seed=5, gain=3.0)
    tc = TA._train_config()
    rec = make_recognizer(cfg, params)
    algo = TA._algorithm(rec, tc)
    ref = {k: np.asarray(v, np.float32).astype(np.float64) for k, v in params.items()}
    ls2 = AN.init_ls2(ref, 1e-2)
    assert AN.noise_name(RO.linear_name(1) + ".W") in algo.noise_parameter_values()
    state = {}
    for step in range(2):
        batch = O.synthetic_batch(cfg, B=3, T=32, seed=100 + step)
        _, eps = TA._replay(algo, step)
        ref, ls2, cost, _, norm = AN.train_step(cfg, ref, ls2, state, batch, tc, eps, TA.N_EXAMPLES, TA.COEF)
        algo.process_batch(dict(zip(algo.SOURCES, batch)))
        assert abs(float(algo.last_cost.item()) - cost) <= 1e-4 * abs(cost), (step, algo.last_cost.item(), cost)
        assert abs(algo.total_gradient_norm() - norm) <= 1e-4 * norm
        got, got_ls2 = rec.get_parameter_values(), algo.noise_parameter_values()
        for k, v in ref.items():
            assert np.abs(got[k] - v).max() <= 1e-4 * np.abs(v).max(), (step, k)
            assert np.abs(got_ls2[AN.noise_name(k)] - ls2[k]).max() <= 1e-4 * np.abs(ls2[k]).max(), (step, k)


def test_compat_train_then_search_with_a_deep_readout(tmp_path, capsys):
    """compat's train (validation and checkpoints included), search and sample from a YAML whose net has
    post_merge_dims: [256, 256] with a Rectifier."""
    _torch()
    import os
    import sys
    import tarfile
    import compat_helpers as CH
    if CH.COMPAT not in sys.path:
        sys.path.insert(0, CH.COMPAT)
    import lvsr.config as C
    import lvsr.main as M
    exp = CH.write_experiment(tmp_path)
    old = "    post_merge_dims: [128]\n    post_merge_activation: !!python/object/apply:blocks.bricks.Maxout [2]\n"
    base = open(exp["base"]).read()
    assert old in base
    open(exp["base"], "w").write(base.replace(
        old, "    post_merge_dims: [256, 256]\n    post_merge_activation: !!python/object/apply:blocks.bricks.Rectifier []\n"))
    cfg = C.Configuration(exp["child"], None, [])
    cfg["cmd_args"] = {}
    save = str(tmp_path / "run")
    M.train_multistage(cfg, save, "", None, "")
    with tarfile.open(os.path.join(save, "main.tar")) as tar:
        names = np.load(__import__("io").BytesIO(tar.extractfile("_parameters").read())).files
    assert "|recognizer|generator|readout|post_merge|mlp|linear_1.W" in names
    capsys.readouterr()
    single = C.Configuration(exp["base"], None, [("monitoring.search.beam_size", "2")])
    decoded = str(tmp_path / "decoded.txt")
    M.search(single, None, os.path.join(save, "main.tar"), "valid", None, None, decoded, False, 1)
    assert "Average CER:" in capsys.readouterr().out
    M.sample(single, None, os.path.join(save, "main.tar"), "valid")
    assert "Utterance 2" in capsys.readouterr().out
