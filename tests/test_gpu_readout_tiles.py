"""The deep readout (net.post_merge_dims of 2 to 4 entries) across the tiles its kernels cut the rows into, against the
float64 oracle of tests/readout_oracle.py.

test_gpu_readout_depth.py runs at most 30 readout rows, so every product of the readout fits in one tile and every
weight gradient is one split.  Here:
  * teacher-forced costs at R = L * B = 1, 127, 128, 129, 304 and 1280 rows, around and across the 128-row tiles of
    gemm_kernel (the merge's and the hidden layers' products with their activation epilogue), on both decoder plans;
  * step-wise log-probabilities at 1 to 300 rows, around and across the 64-row blocks of dense_kernel's DENSE_ACT;
  * full gradients at R = 312 rows (3 row tiles of the forward; gemm_tn's split-K runs several partials through
    tn_reduce_kernel, and readout_bwd_kernel 39 CTAs), at the widest last layer (1408, 48 KB of staged rows) and with
    128 symbols (four logits per lane), and one optimizer step with max-norm;
  * the readout's cost matrix and gradients on the benchmarked training batch (bench.NET, bench.TRAIN_WORKLOAD's
    inputs) over the first 16 of its 64 utterances: 3,040 rows, 24 row tiles;
  * beam search at the widest readout.

The encoder and the decoder's recurrence do not read the readout, so the costs and the benchmark's gradients are
compared with the oracle applied to the GPU's own encoder output.  The gradient tests run the whole model in float64
(RO.cost_and_grads).  Rectifier readouts are first moved off their kinks (RO.clear_kinks): a pre-activation within
float32 error of 0 may take either side of the derivative's jump.  Bars, those of test_gpu_readout_depth.py: costs to
2e-4 of max(1, |want|), the cost to 1e-4, gradients to 1e-4 of each parameter's largest entry plus 1e-6 of the model's
largest.  Every test prints its worst error over its bar."""
from collections import OrderedDict

import numpy as np
import pytest

import bench
import content_oracle as CO
import readout_oracle as RO
from helpers import O, f32, make_recognizer, package
from oracle import lvsr_oracle_grad as G

pytestmark = pytest.mark.gpu

MLP = RO.PM + "/mlp/"
KINK = 1e-4          # the kink screen's band: well above the float32 error of a readout pre-activation


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _cfg(dims, act, V, attention="content_and_conv", use_states=True):
    base = dict(num_features=40, dims_bidir=[128], subsample=[1], dim_dec=128, dim_matcher=128, conv_n=8,
                conv_num_filters=4, num_phonemes=V, post_merge_dims=dims[:1], post_merge_activation=act,
                maxout_pieces=1, use_states_for_readout=use_states, max_decoded_length_scale=2.0)
    cfg = CO.make_config(**base) if attention == "content" else O.make_config(**base)
    cfg["post_merge_dims"] = [int(d) for d in dims]
    return cfg


def _params(cfg, seed=3, gain=10.0):
    """float32 parameters with the deep MLP, weights large enough that every layer matters (as
    test_gpu_readout_depth._params draws them)."""
    mod = CO if cfg.get("attention_type") == "content" else O
    base = mod.init_params(dict(cfg, post_merge_dims=cfg["post_merge_dims"][:1]), seed=seed, scale=gain)
    rng = np.random.RandomState(seed + 100)
    dims, V = cfg["post_merge_dims"], cfg["num_phonemes"]
    out = OrderedDict()
    for k, v in base.items():
        if k.startswith(MLP):
            continue
        out[k] = f32(v)
        if k == RO.PM + "/bias.b":
            for j in range(len(dims)):
                din, dout = dims[j], dims[j + 1] if j + 1 < len(dims) else V
                out[RO.linear_name(j) + ".b"] = f32(rng.normal(0, 0.3, size=(dout,)))
                out[RO.linear_name(j) + ".W"] = f32(rng.normal(0, 1.5 / np.sqrt(din), size=(din, dout)))
    return out


def _encode(rec, x, m):
    att, attm = rec.encode(x, m)
    return att, attm, f32(att.cpu().numpy()), f32(attm.cpu().numpy())


def _decoder(cfg):
    return CO if cfg.get("attention_type") == "content" else O


def _oracle_costs(cfg, params, att, attm, labels, lmask):
    """The oracle's teacher-forced costs of the deep model from the attended sequence."""
    r = _decoder(cfg).cost_matrix(cfg, RO.shallow_params(cfg, params), att, attm, labels, lmask, return_all=True)
    logits = RO.readout(cfg, params, r["states"], r["weighted_averages"])
    return -np.take_along_axis(O.log_softmax(logits), labels[..., None], axis=-1)[..., 0] * lmask


def _cost_err(got, want):
    """worst |got - want| over the costs' bar, 2e-4 of max(1, |want|)"""
    return float(np.abs(got - want).max() / (2e-4 * max(1.0, np.abs(want).max())))


def _labels(cfg, B, L, seed):
    """labels [L, B] with one utterance of all L steps and the others of ceil(L/2) .. L, each ending in eos; the
    masked tail rows hold random symbols too"""
    rng = np.random.RandomState(seed)
    V = cfg["num_phonemes"]
    n = rng.randint(-(-L // 2), L + 1, size=B)
    n[rng.randint(B)] = L
    labels = rng.randint(0, V - 1, size=(L, B)).astype(np.int64)
    labels[n - 1, np.arange(B)] = cfg["eos_label"]
    lmask = (np.arange(L)[:, None] < n[None, :]).astype(np.float64)
    return labels, lmask


def _recordings(cfg, B, T, seed):
    rng = np.random.RandomState(seed)
    lens = rng.randint(-(-3 * T // 5), T + 1, size=B)
    lens[rng.randint(B)] = T
    m = (np.arange(T)[:, None] < lens[None, :]).astype(np.float64)
    return rng.normal(size=(T, B, cfg["num_features"])) * m[:, :, None], m


# ---- 1. teacher-forced rows across gemm_kernel's 128-row tiles ------------------------------------------------------

# (B, L) with R = L * B = 1, 127, 128, 129, 304, 1280; last widths below one 128-column tile (8), across tiles (136)
# and the widest (1408); every activation at depths 2 to 4; V of 5, 97 (not a multiple of 4) and 128
TF_CASES = [
    (1, 1, [8, 136], "relu", 5),
    (1, 127, [136, 8], "tanh", 97),
    (2, 64, [128, 1408], "identity", 128),
    (3, 43, [136, 136, 136], "maxout", 97),
    (16, 19, [256, 8, 1408], "relu", 128),
    (16, 19, [1408, 136], "maxout", 5),
    (64, 20, [8, 136, 72, 1408], "tanh", 5),
    (64, 20, [136, 1408, 8], "relu", 97),
]


@pytest.mark.parametrize("B,L,dims,act,V", TF_CASES)
@pytest.mark.parametrize("stepwise", [False, True])
def test_teacher_forced_rows_across_tiles(B, L, dims, act, V, stepwise, monkeypatch):
    _torch()
    if stepwise:
        monkeypatch.setenv("LVSR_NO_DEC_SCAN", "1")
    cfg = _cfg(dims, act, V)
    params = _params(cfg, seed=B + L)
    rec = make_recognizer(cfg, params)
    x, m = _recordings(cfg, B, 24, seed=L)
    labels, lmask = _labels(cfg, B, L, seed=B)
    att, attm, att64, attm64 = _encode(rec, x, m)
    got = rec.cost_matrix(labels, lmask, att, attm).cpu().numpy()
    plan = rec.decoder_plan()
    want = _oracle_costs(cfg, params, att64, attm64, labels, lmask)
    err = _cost_err(got, want)
    print("R = %d, decoder %s: worst cost error / bar %.2e" % (L * B, plan.get("kernel"), err))
    assert err <= 1.0
    assert not got[lmask == 0].any()
    assert plan["ran"] == (not stepwise), plan


# ---- 2. step-wise rows across dense_kernel's 64-row blocks ----------------------------------------------------------

@pytest.mark.parametrize("dims,act,V", [([136, 8], "relu", 128), ([128, 1408], "tanh", 97),
                                        ([72, 8, 1408], "maxout", 128)])
@pytest.mark.parametrize("R", [1, 63, 64, 65, 128, 300])
def test_stepwise_logprobs_across_row_blocks(dims, act, V, R):
    """R hypotheses over up to three utterances, advanced one or two steps by random symbols so that every row differs,
    then lvsr_logprobs against RO.logprobs_computer at the GPU's own states."""
    torch = _torch()
    cfg = _cfg(dims, act, V)
    params = _params(cfg, seed=R)
    rec = make_recognizer(cfg, params)
    U = min(R, 3)
    x, m, _, _ = O.synthetic_batch(cfg, B=U, T=40, seed=R + 1)
    att, attm, att64, attm64 = _encode(rec, x, m)
    ru = np.arange(R) % U
    ctx = dict(attended=att, attended_mask=attm, preprocessed=rec.preprocess(att),
               row_utt=torch.as_tensor(ru.astype(np.int32), device=att.device))
    st = rec._initial_states(att.shape[0], R)
    rng = np.random.RandomState(R)
    for _ in range(1 + R % 2):
        st = rec._next_states(ctx, st, rng.randint(0, V, size=R))
    got = rec._logprobs(ctx, st).cpu().numpy()
    ost = {k: f32(v.cpu().numpy()) if v.dtype == torch.float32 else v.cpu().numpy() for k, v in st.items()}
    want = RO.logprobs_computer(cfg, params, att64[:, ru], attm64[:, ru], ost)
    assert R < 2 or np.abs(want[1:] - want[:-1]).max() > 1e-3          # the rows differ
    err = _cost_err(got, want)
    print("R = %d: worst log-probability error / bar %.2e" % (R, err))
    assert err <= 1.0


# ---- 3. full gradients at a few hundred rows ------------------------------------------------------------------------

GRAD_CASES = {
    "tanh_1408_V128": ([128, 1408], "tanh", 128, "content_and_conv", True),
    "relu_1408_V128": ([128, 1408], "relu", 128, "content_and_conv", True),
    "identity_256_8_1408_V97": ([256, 8, 1408], "identity", 97, "content_and_conv", True),
    "relu_128_72_72_8_V5": ([128, 72, 72, 8], "relu", 5, "content_and_conv", True),
    "maxout1_depth3_no_states": ([136, 256, 72], "maxout", 32, "content_and_conv", False),
    "relu_depth2_content": ([128, 256], "relu", 32, "content", True),
}


def _grad_setup(name, seed=7):
    """(cfg, params moved off their kinks, batch of B = 8 utterances of up to 300 frames: L = 39, R = 312)"""
    dims, act, V, attention, use_states = GRAD_CASES[name]
    cfg = _cfg(dims, act, V, attention, use_states)
    params = _params(cfg, seed=seed, gain=3.0)
    for k in params:
        if k.startswith(O._GEN + "/readout/merge/"):
            params[k] = f32(params[k] * 100.0)         # h_0's pre-activations of order 1, where tanh and relu bend
    batch = O.synthetic_batch(cfg, B=8, T=300, seed=12)
    assert batch[2].size == 312
    r = _decoder(cfg).recognizer_cost(cfg, RO.shallow_params(cfg, params), *batch, return_all=True)
    params, moved = RO.clear_kinks(cfg, params, r["states"], r["weighted_averages"], batch[3] > 0, KINK)
    if moved:
        print("%d Rectifier units moved off their kinks by at most %.1e" % (len(moved), max(abs(s) for *_, s in moved)))
    return cfg, params, batch


@pytest.mark.parametrize("name", list(GRAD_CASES))
def test_gradients_at_hundreds_of_rows(name):
    _torch()
    pkg = package()
    cfg, params, batch = _grad_setup(name)
    rec = make_recognizer(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
    cost, grads = algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
    want_cost, want = RO.cost_and_grads(cfg, params, *batch)
    assert set(grads) == set(want)
    gmax = max(np.abs(w).max() for w in want.values())
    errs = {k: float(np.abs(grads[k] - w).max() / (1e-4 * np.abs(w).max() + 1e-6 * gmax)) for k, w in want.items()}
    worst = max(errs, key=errs.get)
    cost_err = abs(cost - want_cost) / (1e-4 * abs(want_cost))
    print("cost error / bar %.2e; worst gradient error / bar %.2e (%s)" % (cost_err, errs[worst], worst))
    assert cost_err <= 1.0
    assert not {k: e for k, e in errs.items() if e > 1.0}, errs


def test_optimizer_step_with_max_norm_at_the_widest_readout():
    _torch()
    pkg = package()
    cfg, params, batch = _grad_setup("tanh_1408_V128")
    tc = G.make_train_config(gradient_threshold=2.0, rules=("momentum", "adadelta"), scale=0.05, momentum=0.5,
                             decay_rate=0.95, epsilon=1e-6, max_norm=1.0)
    rec = make_recognizer(cfg, params)
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(tc, dict(max_norm=1.0)))
    algo.initialize()
    ref, ref_cost, _ = RO.train_step(cfg, params, {}, batch, tc)
    algo.process_batch(dict(zip(algo.SOURCES, batch)))
    cost_err = abs(float(algo.last_cost.item()) - ref_cost) / (1e-4 * abs(ref_cost))
    got = rec.get_parameter_values()
    errs = {k: float(np.abs(got[k] - v).max() / (2e-5 * max(1.0, np.abs(v).max()) + 1e-6)) for k, v in ref.items()}
    worst = max(errs, key=errs.get)
    print("cost error / bar %.2e; worst parameter error / bar %.2e (%s)" % (cost_err, errs[worst], worst))
    assert cost_err <= 1.0
    assert not {k: e for k, e in errs.items() if e > 1.0}, errs
    for j in range(2):
        W = got[RO.linear_name(j) + ".W"].astype(np.float64)
        assert (np.sqrt((W ** 2).sum(axis=0)) <= 1.0 + 1e-5).all(), j
    # max-norm bound the widest layer: its columns were longer than 1 before the step
    assert (np.sqrt((params[RO.linear_name(0) + ".W"].astype(np.float64) ** 2).sum(axis=0)) > 1.0).any()


# ---- 4. the benchmark's training batch ------------------------------------------------------------------------------

BENCH_READOUTS = {"tanh_256x2": ([256, 256], "tanh"), "identity_256x3": ([256, 256, 256], "identity")}
# of bench.train_bench's 64 utterances: the numpy decoder's 190 steps take about 25 s over these 16 and over two
# minutes over all 64
BENCH_UTTS = 16


def _bench_model(dims, act):
    pkg = package()
    W, N = bench.TRAIN_WORKLOAD, bench.NET
    net = {k: v for k, v in N.items() if k not in ("post_merge_dims", "maxout_pieces")}
    cfg = RO.make_config(dims, post_merge_activation=act, maxout_pieces=1, eos_label=W["V"] - 1, **net)
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": W["F"]}, input_num_chars={}, eos_label=W["V"] - 1, num_phonemes=W["V"],
        dim_dec=N["dim_dec"], dims_bidir=N["dims_bidir"], subsample=N["subsample"], conv_n=N["conv_n"],
        conv_num_filters=N["conv_num_filters"], dim_matcher=N["dim_matcher"], post_merge_dims=dims,
        post_merge_activation=pkg.Tanh() if act == "tanh" else pkg.Identity(), enc_transition=pkg.GatedRecurrent,
        dec_transition=pkg.GatedRecurrent)
    assert list(rec.parameter_shapes().items()) == list(RO.param_shapes(cfg).items())
    return cfg, rec


@pytest.fixture(scope="module")
def bench_decoder():
    """The first BENCH_UTTS utterances of bench.train_bench's batch, the [256, 256] model's parameters from
    bench.init_values, the GPU's encoder output of that batch and the oracle decoder's states and glimpses on it."""
    _torch()
    cfg, rec = _bench_model([256, 256], "tanh")
    params = bench.init_values(RO.param_shapes(cfg), seed=1)
    rec.set_parameter_values(params)
    x, m, labels, lm = bench.synthetic_batch(**bench.TRAIN_WORKLOAD, seed=bench.shard_seed(0, base=4321))
    batch = (x[:, :BENCH_UTTS], m[:, :BENCH_UTTS], labels[:, :BENCH_UTTS], lm[:, :BENCH_UTTS])
    assert batch[2].size == 190 * BENCH_UTTS
    _, _, att64, attm64 = _encode(rec, batch[0], batch[1])
    p64 = OrderedDict((k, np.asarray(v, np.float64)) for k, v in params.items())
    r = O.cost_matrix(cfg, RO.shallow_params(cfg, p64), att64, attm64, batch[2], batch[3].astype(np.float64),
                      return_all=True)
    return params, batch, att64, r["states"], r["weighted_averages"]


@pytest.mark.parametrize("name", list(BENCH_READOUTS))
def test_readout_on_the_benchmarked_training_batch(name, bench_decoder):
    """The cost matrix and the readout family's gradients of one cost_and_gradients call against a float64 restatement
    of the readout on the oracle decoder's states and glimpses.  The decoder never reads the readout, so this checks
    those gradients in full; the gradients below the readout are test_gpu_bench_train.py's (depth 1) and
    test_gradients_at_hundreds_of_rows' (deep)."""
    torch = _torch()
    pkg = package()
    base, batch, att64, states, ctx = bench_decoder
    dims, act = BENCH_READOUTS[name]
    cfg, rec = _bench_model(dims, act)
    values = bench.init_values(RO.param_shapes(cfg), seed=1)
    params = OrderedDict((k, values[k] if k.startswith(MLP) else base[k]) for k in values)
    rec.set_parameter_values(params)
    labels, lm = batch[2], batch[3]
    att, attm, a64, _ = _encode(rec, batch[0], batch[1])
    assert np.array_equal(a64, att64)          # the same encoder output the oracle's decoder ran on
    got_costs = rec.cost_matrix(labels, lm, att, attm).cpu().numpy()
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]))
    cost, grads = algo.cost_and_gradients(dict(zip(algo.SOURCES, batch)))
    names = [k for k in params if k.startswith(RO.PM + "/") or k.startswith(O._GEN + "/readout/merge/")]
    assert len(names) == 1 + 2 * len(dims) + 2
    p = OrderedDict((k, torch.tensor(np.asarray(params[k], np.float64), requires_grad=True)) for k in names)
    logits = RO.readout_torch(cfg, p, torch.as_tensor(states), torch.as_tensor(ctx))
    logp = torch.log_softmax(logits, dim=-1)
    costs = -torch.gather(logp, 2, torch.as_tensor(labels)[..., None])[..., 0] * torch.as_tensor(lm.astype(np.float64))
    want_cost = costs.sum() / labels.shape[1]
    want = dict(zip(names, (g.numpy() for g in torch.autograd.grad(want_cost, list(p.values())))))
    want_costs, want_cost = costs.detach().numpy(), float(want_cost.detach())
    gmax = max(np.abs(w).max() for w in want.values())
    errs = {k: float(np.abs(grads[k] - w).max() / (1e-4 * np.abs(w).max() + 1e-6 * gmax)) for k, w in want.items()}
    worst = max(errs, key=errs.get)
    cerr, cost_err = _cost_err(got_costs, want_costs), abs(cost - want_cost) / (1e-4 * abs(want_cost))
    print("R = %d: cost matrix error / bar %.2e, cost %.2e, worst gradient error / bar %.2e (%s)" % (
        labels.size, cerr, cost_err, errs[worst], worst))
    assert cerr <= 1.0 and cost_err <= 1.0
    assert not {k: e for k, e in errs.items() if e > 1.0}, errs


# ---- 5. beam search at the widest readout ---------------------------------------------------------------------------

def test_beam_search_at_the_widest_readout():
    _torch()
    cfg = _cfg([128, 1408], "tanh", 128)
    params = _params(cfg, seed=9)
    params[RO.linear_name(1) + ".b"][cfg["eos_label"]] += 3.0
    rec = make_recognizer(cfg, params)
    rng = np.random.RandomState(5)
    utts = [rng.normal(size=(T, cfg["num_features"])) for T in (40, 27, 33)]
    rec.init_beam_search(10)
    got = rec.beam_search_many([{"recordings": u} for u in utts], raise_on_failure=False)
    found, worst = 0, 0.0
    for u, g in zip(utts, got):
        try:
            want = RO.beam_search(cfg, params, u, 10)
        except O.CandidateNotFoundError:
            assert g is None
            continue
        found += 1
        assert g is not None and g[0] == want[0]
        gc, wc = np.asarray(g[1], np.float64), np.asarray(want[1], np.float64)
        worst = max(worst, float((np.abs(gc - wc) / (5e-3 + 1e-3 * np.abs(wc))).max()))
    print("%d of 3 found; worst search cost error / bar %.2e" % (found, worst))
    assert found >= 1 and worst <= 1.0
