"""The training loop of lvsr/main.py on the GPU: adaptive clipping inside the update against the float64 oracles fed
the restated thresholds (with and without adaptive noise), its launch count and stream behaviour, the alignment
statistics kernel against numpy, and a compat multi-stage run with validation, search, patience and restart_from."""
import os
import sys

import numpy as np
import pytest

import adaptive_noise_oracle as AN
import content_oracle as CO
import training_loop_oracle as TL
from compat_helpers import COMPAT, write_experiment
from helpers import O, PYRAMID, make_recognizer, package
from oracle import lvsr_oracle_grad as G

pytestmark = pytest.mark.gpu

THR0, BURNIN, DECAY = 20.0, 3, 0.9
TC = G.make_train_config(gradient_threshold=THR0, rules=("momentum", "adadelta"), scale=0.05, momentum=0.5,
                         decay_rate=0.95, epsilon=1e-6, max_norm=1.0)
N_EXAMPLES, COEF = 40, 0.5
NOISE_THR0 = 1e-3          # under adaptive noise every step is clipped: at thr0, then at the cap 5 thr0


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _algorithm(rec, adaptive=True, noise=False, tc=TC):
    pkg = package()
    rule = pkg.step_rule_from_config(tc, dict(max_norm=tc["max_norm"]))
    if noise:          # a log-variance step of the size an unclipped one takes makes the noise, and the cost, explode
        pkg.clipping_rule(rule).threshold = NOISE_THR0
    if adaptive:
        pkg.adaptive_clipping(rule, burnin_period=BURNIN, decay_rate=DECAY)
    an = dict(num_examples=N_EXAMPLES, init_sigma=1e-2, model_cost_coefficient=COEF, seed=7) if noise else None
    algo = pkg.GradientDescent(recognizer=rec, step_rule=rule, adaptive_noise=an)
    algo.initialize()
    return algo, pkg.clipping_rule(rule)


def _replay(algo, update):
    torch = _torch()
    rec = algo.recognizer
    lib, h = package()._lib.load(), rec._require_ready()
    buf = torch.zeros((algo._n,), dtype=torch.float32, device=rec.device)
    package()._lib.check(lib.lvsr_train_noise_sample(h, update, buf.data_ptr(), rec._stream()))
    flat = buf.cpu().numpy()
    shapes = rec.parameter_shapes()
    return {k: flat[o:o + c].reshape(shapes[k]).astype(np.float64) for k, (o, c) in algo._offsets().items()}


@pytest.mark.parametrize("noise", [False, True], ids=["plain", "adaptive_noise"])
def test_adaptive_clipping_matches_the_oracle(noise):
    """8 updates, burn-in 3, decay 0.9.  Without noise, thr0 20: the first steps are unclipped, the later ones clipped
    by the adaptive threshold.  Each oracle step clips with the threshold the restatement derives from the oracle's
    norms; the device's threshold is the restatement's on the device's norms to 1e-6."""
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    rec = make_recognizer(cfg, params)
    algo, clip = _algorithm(rec, noise=noise)
    thr0 = NOISE_THR0 if noise else THR0
    ref = {k: np.asarray(v, np.float32).astype(np.float64) for k, v in params.items()}
    ls2 = AN.init_ls2(ref, 1e-2) if noise else None
    on_oracle = TL.AdaptiveClipping(thr0, BURNIN, DECAY)
    on_device = TL.AdaptiveClipping(thr0, BURNIN, DECAY)
    state, clipped = {}, []
    for step in range(8):
        batch = O.synthetic_batch(cfg, B=4, T=40, seed=100 + step)
        got_thr = clip.current_threshold()
        assert abs(got_thr - on_device.threshold) <= 1e-6 * on_device.threshold, (step, got_thr, on_device.threshold)
        tc = dict(TC, gradient_threshold=on_oracle.threshold)
        if noise:
            eps = _replay(algo, step)
            ref, ls2, cost, _, norm = AN.train_step(cfg, ref, ls2, state, batch, tc, eps, N_EXAMPLES, COEF)
        else:
            ref, cost, grads = G.train_step(cfg, ref, state, batch, tc)
            norm = G.l2_norm(grads.values())
        clipped.append(norm >= on_oracle.threshold)
        algo.process_batch(dict(zip(algo.SOURCES, batch)))
        got_norm = algo.total_gradient_norm()
        assert abs(got_norm - norm) <= 1e-4 * norm, (step, got_norm, norm)
        assert abs(float(algo.last_cost.item()) - cost) <= 1e-4 * abs(cost), (step, cost)
        on_oracle.after_batch(float(np.float32(norm)))
        on_device.after_batch(got_norm)
        got = rec.get_parameter_values()
        for k, v in ref.items():
            if noise:
                assert np.abs(got[k] - v).max() <= 1e-4 * np.abs(v).max(), (step, k)
            else:
                assert np.abs(got[k] - v).max() <= 2e-5 * max(1.0, np.abs(v).max()) + 1e-6, (step, k)
        if noise:
            got_ls2 = algo.noise_parameter_values()
            for k, w in ls2.items():
                assert np.abs(got_ls2[AN.noise_name(k)] - w).max() <= 1e-4 * np.abs(w).max(), (step, k)
    print("clipped steps:", clipped)
    if noise:
        assert all(clipped), clipped
    else:
        assert any(clipped) and not all(clipped), clipped
    # lvsr_train_reset (GradientDescent.initialize) puts the state back to thr0
    algo.initialize()
    assert clip.current_threshold() == thr0


def test_adaptive_clipping_adds_no_launch():
    _torch()
    pkg = package()
    lib = pkg._lib.load()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    counts = {}
    for adaptive in (False, True):
        rec = make_recognizer(cfg, params)
        algo, _ = _algorithm(rec, adaptive=adaptive)
        for step in range(2):                    # the first step sizes workspaces and allocates optimizer state
            batch = dict(zip(algo.SOURCES, O.synthetic_batch(cfg, B=4, T=40, seed=100 + step)))
            lib.lvsr_launch_count(1)
            algo.process_batch(batch)
            counts[adaptive, step] = int(lib.lvsr_launch_count(0))
    assert counts[True, 1] == counts[False, 1], counts


def test_process_batch_does_not_wait_for_the_stream():
    """A spin queued on a non-blocking stream is still running when process_batch returns with adaptive clipping on:
    the update reads and writes its threshold on the device, without a host round trip."""
    torch = _torch()
    from test_gpu_streams import SPIN, _side_stream
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    rec = make_recognizer(cfg, params)
    algo, clip = _algorithm(rec)
    s = _side_stream()
    batches = [dict(zip(algo.SOURCES, [None if a is None else torch.as_tensor(np.ascontiguousarray(a), device="cuda")
                                       for a in O.synthetic_batch(cfg, B=4, T=40, seed=100 + i)])) for i in range(2)]
    s.wait_stream(torch.cuda.default_stream())
    with torch.cuda.stream(s):
        algo.process_batch(batches[0])           # warm-up: sizes the workspaces on s
        n1 = algo.total_gradient_norm()          # (synchronises)
        torch.cuda._sleep(SPIN)
        algo.process_batch(batches[1])
        pending = not s.query()
    assert pending
    n2 = algo.total_gradient_norm()
    want = TL.AdaptiveClipping(THR0, BURNIN, DECAY)
    want.after_batch(n1)
    want.after_batch(n2)
    got = clip.current_threshold()
    assert abs(got - want.threshold) <= 1e-6 * want.threshold, (got, want.threshold)


def _softmax_rows(rng, L, B, Tp, peaky=8.0):
    e = rng.normal(size=(L, B, Tp)) * peaky
    w = np.exp(e - e.max(-1, keepdims=True))
    return (w / w.sum(-1, keepdims=True)).astype(np.float32)


@pytest.mark.parametrize("B,Tp", [(1, 7), (37, 300), (64, 2000)])
def test_alignment_statistics_kernel_matches_numpy(B, Tp):
    torch = _torch()
    cfg = O.make_config(**PYRAMID)
    rec = make_recognizer(cfg, O.init_params(cfg, seed=1))
    rng = np.random.RandomState(B)
    L = 23
    w = _softmax_rows(rng, L, B, Tp)
    w[:, :, Tp // 2:] *= (rng.uniform(size=(L, B, 1)) < 0.3)        # some rows end early: zeros in the tail
    mask = (np.arange(L)[:, None] < rng.randint(1, L + 1, size=B)[None, :]).astype(np.float32)
    out = torch.zeros((2,), dtype=torch.float64, device="cuda")
    for m in (None, mask):
        rec.alignment_statistics(torch.as_tensor(w, device="cuda"), None if m is None else torch.as_tensor(m, device="cuda"),
                                 out)
        got = out.cpu().numpy()
        want = TL.alignment_stats(w, m)
        assert abs(got[0] - want[0]) <= 1e-5 * abs(want[0]), (got, want)
        assert abs(got[1] - want[1]) <= 1e-5 * abs(want[1]) + 1e-12, (got, want)
        again = out.clone()
        rec.alignment_statistics(torch.as_tensor(w, device="cuda"), None if m is None else torch.as_tensor(m, device="cuda"),
                                 out)
        assert torch.equal(again, out)                                  # a fixed order of summation


PRIORS = [None, dict(type="window_around_median", before=5, after=7),
          dict(type="expanding", initial_begin=0, initial_end=6, min_speed=0.7, max_speed=2.2)]


@pytest.mark.parametrize("case", ["default", "window_around_median", "expanding", "content"])
def test_validation_statistics_of_a_batch(case):
    """SpeechRecognizer.validation_statistics on a masked batch: the cost is the oracle's summed cost matrix and the
    two sums are numpy's on the weights lvsr_cost_matrix returns."""
    torch = _torch()
    if case == "content":
        cfg = CO.make_config(num_features=40, dims_bidir=[128], subsample=[1], dim_dec=128, dim_matcher=128,
                             num_phonemes=32, post_merge_dims=[128], maxout_pieces=2)
        params = CO.init_params(cfg, seed=3, scale=10.0)
        cost_fn = CO.recognizer_cost
    else:
        prior = PRIORS[["default", "window_around_median", "expanding"].index(case)]
        cfg = O.make_config(prior=prior, **PYRAMID)
        params = O.init_params(cfg, seed=3, scale=10.0)
        cost_fn = O.recognizer_cost
    rec = make_recognizer(cfg, params)
    x, m, labels, lm = O.synthetic_batch(cfg, B=5, T=48, seed=11)
    s = rec.validation_statistics(x, m, labels, lm)
    costs = rec.cost(x, m, labels, lm).astype(np.float64)
    assert abs(s["cost"] - costs.sum()) <= 1e-5 * abs(costs.sum())
    want = cost_fn(cfg, params, x, m, labels, lm).sum()
    assert abs(s["cost"] - want) <= 1e-4 * abs(want)
    att, attm = rec.encode(x, m)
    w = rec.cost_matrix(labels, lm, att, attm, return_all=True)["weights"].cpu().numpy()
    ent, pen = TL.alignment_stats(w, lm)
    assert abs(s["weights_entropy"] - ent) <= 1e-5 * abs(ent)
    assert abs(s["weights_penalty"] - pen) <= 1e-5 * abs(pen) + 1e-9
    assert s["num_labels"] == float(lm.sum()) and s["batch_size"] == 5


MULTISTAGE = """
parent: {base}
data:
    validation_batch_size: 2
training:
    num_epochs: 6
    patience:
        min_epochs: 2
        patience_factor: 1.5
monitoring:
    validate_every_epochs: 1
    search_every_epochs: 1
stages:
    pretraining:
        number: 0
        training:
            num_epochs: 6
    main:
        number: 1
        training:
            num_epochs: 1
            restart_from: _best_ll
"""


def test_compat_multistage_with_validation_patience_and_restart_from(tmp_path, monkeypatch):
    _torch()
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as LC
    import lvsr.main as M
    exp = write_experiment(tmp_path)
    path = os.path.join(str(tmp_path), "multistage.yaml")
    with open(path, "w") as f:
        f.write(MULTISTAGE.format(base=exp["base"]))
    cfg = LC.Configuration(path, None, [])
    made = []
    real_create = M.create_model

    def create_model(config, data, load_path=None, test_tag=False):
        rec = real_create(config, data, load_path, test_tag)
        made.append((load_path, rec, rec.get_parameter_values()))
        return rec

    monkeypatch.setattr(M, "create_model", create_model)
    out = str(tmp_path / "run")
    M.train_multistage(cfg, out, "", None, None)
    (pre_path, pre, _), (main_path, main, main_start) = made
    assert pre_path is None and main_path == os.path.join(out, "pretraining_best_ll.tar")
    best = package().SpeechRecognizer.load_checkpoint_values(main_path)
    for k, v in main_start.items():
        assert np.array_equal(v, best[k]), k
    # the stop epoch of pretraining follows from its logged records
    log = pre.training_log
    epochs = log.status["epochs_done"]
    rows = [log.rows[0]] + [log.rows[e * 3] for e in range(1, epochs + 1)]         # 10 utterances: 3 batches per epoch
    notified = set(TL.track_the_best([r["valid_sequence_total_cost"] for r in rows])) | \
        set(TL.track_the_best([r["valid_per"] for r in rows]))
    stop = TL.patience_stop_epoch(notified - {0}, 2, 1.5, 6)
    assert epochs == (stop or 6), (epochs, stop, rows)
    files = set(os.listdir(out))
    assert {"pretraining.tar", "pretraining_best_ll.tar", "main.tar"} <= files <= {
        "pretraining.tar", "pretraining_best_ll.tar", "pretraining_best.tar", "main.tar", "main_best_ll.tar",
        "main_best.tar"}, files
    # PER through beam_search_many equals the per-utterance beam search
    data = M.Data(**cfg["data"])
    search = cfg["monitoring"]["search"]
    per = M.phoneme_error_rate(main, data, **search)
    errors = length = 0.0
    kw = dict(char_discount=search["char_discount"], round_to_inf=search["round_to_inf"], stop_on=search["stop_on"])
    kw = {k: v for k, v in kw.items() if v}
    for ex in data.examples("valid"):
        truth = data.info_dataset.decode(ex["labels"])
        try:
            outputs, _ = main.beam_search({"recordings": ex["recordings"]}, **kw)
            err = min(1, M.wer(truth, data.info_dataset.decode(outputs[0])))
        except M.CandidateNotFoundError:
            err = 1.0
        errors += err * len(truth)
        length += len(truth)
    assert per == pytest.approx(errors / length, abs=1e-12)
    # main's validation before its first epoch sees pretraining's best-ll parameters
    best_epoch = max(TL.track_the_best([r["valid_sequence_total_cost"] for r in rows]))
    assert main.training_log.rows[0]["valid_sequence_total_cost"] == pytest.approx(
        rows[best_epoch]["valid_sequence_total_cost"], rel=1e-5)
