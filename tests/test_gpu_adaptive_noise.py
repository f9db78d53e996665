"""Adaptive weight noise on the GPU (regularization.adaptive_noise; lvsr/graph.py:71-251, include/lvsr_b200.h):
the replayed eps against N(0, 1), one and two training steps against the float64 oracle
(tests/adaptive_noise_oracle.py) given that eps, inference on the means, determinism, the "noise" profile class, and
a three-stage compat run."""
import ctypes as C
import io
import logging
import os
import sys
import tarfile

import numpy as np
import pytest

import adaptive_noise_oracle as AN
import content_oracle as CO
from compat_helpers import COMPAT, write_experiment
from helpers import O, PYRAMID, make_recognizer, package
from oracle import lvsr_oracle_grad as G

pytestmark = pytest.mark.gpu

N_EXAMPLES, COEF = 40, 0.5


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _train_config(threshold=2.0, rules=("momentum", "adadelta"), max_norm=1.0, scale=0.05):
    return G.make_train_config(gradient_threshold=threshold, rules=rules, scale=scale, momentum=0.5, decay_rate=0.95,
                               epsilon=1e-6, max_norm=max_norm)


def _algorithm(rec, tc, init_sigma=1e-2, seed=7):
    pkg = package()
    algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(tc, dict(max_norm=tc["max_norm"])),
                               adaptive_noise=dict(num_examples=N_EXAMPLES, init_sigma=init_sigma,
                                                   model_cost_coefficient=COEF, seed=seed))
    algo.initialize()
    return algo


def _replay(algo, update):
    """(flat eps of `update`, {parameter name: eps})."""
    torch = _torch()
    rec = algo.recognizer
    lib, h = package()._lib.load(), rec._require_ready()
    buf = torch.full((algo._n,), 7.0, dtype=torch.float32, device=rec.device)
    package()._lib.check(lib.lvsr_train_noise_sample(h, update, buf.data_ptr(), rec._stream()))
    flat = buf.cpu().numpy()
    shapes = rec.parameter_shapes()
    return flat, {k: flat[o:o + c].reshape(shapes[k]).astype(np.float64) for k, (o, c) in algo._offsets().items()}


def _inside(algo):
    mask = np.zeros(algo._n, bool)
    for o, c in algo._offsets().values():
        mask[o:o + c] = True
    return mask


def test_eps_is_standard_normal_fresh_per_update_and_seed_and_the_padding_stays_zero():
    from scipy import stats
    _torch()
    cfg = O.make_config(**PYRAMID)
    rec = make_recognizer(cfg, O.init_params(cfg, seed=5, scale=10.0))
    algo = _algorithm(rec, _train_config())
    inside = _inside(algo)
    flat0, _ = _replay(algo, 0)
    flat1, _ = _replay(algo, 1)
    assert not flat0[~inside].any() and not flat1[~inside].any()
    e0, e1 = flat0[inside].astype(np.float64), flat1[inside].astype(np.float64)
    n = e0.size
    assert abs(e0.mean()) < 5 / np.sqrt(n) and abs(e0.var() - 1) < 5 * np.sqrt(2.0 / n), (e0.mean(), e0.var())
    assert stats.kstest(e0, "norm").pvalue > 1e-4 and stats.kstest(e1, "norm").pvalue > 1e-4
    assert abs(np.corrcoef(e0, e1)[0, 1]) < 5 / np.sqrt(n)
    # neighbouring elements (the four normals of one Philox call) are uncorrelated too
    assert abs(np.corrcoef(e0[:-1], e0[1:])[0, 1]) < 5 / np.sqrt(n)
    other = _algorithm(make_recognizer(cfg, O.init_params(cfg, seed=5, scale=10.0)), _train_config(), seed=8)
    e_seed = _replay(other, 0)[0][inside].astype(np.float64)
    assert abs(np.corrcoef(e0, e_seed)[0, 1]) < 5 / np.sqrt(n)
    # the buffer the training forward ran on: p + eps exp(1024 ls2) inside the parameters, exact zeros in the padding
    torch = _torch()
    means = rec.get_parameter_values()
    sigma = np.exp(1024.0 * float(AN.init_ls2({"x": np.zeros(1)}, 1e-2)["x"][0]))
    algo.cost_and_gradients(dict(zip(algo.SOURCES, O.synthetic_batch(cfg, B=2, T=24, seed=3))))
    buf = torch.full((algo._n,), 7.0, dtype=torch.float32, device=rec.device)
    package()._lib.check(package()._lib.load().lvsr_train_noise_params(rec._require_ready(), buf.data_ptr(), rec._stream()))
    noisy = buf.cpu().numpy()
    assert not noisy[~inside].any()
    for k, (o, c) in algo._offsets().items():
        p = means[k].reshape(-1).astype(np.float64)
        want = p + flat0[o:o + c].astype(np.float64) * sigma
        err = np.abs(noisy[o:o + c] - want)
        assert (err <= 2e-7 * np.abs(want) + 1e-6 * sigma * np.abs(flat0[o:o + c])).all(), (k, err.max())


def _cases():
    timit = dict(num_features=123, dims_bidir=[128, 128], subsample=[1, 2], dim_dec=128, dim_matcher=128,
                 num_phonemes=63, post_merge_dims=[128], maxout_pieces=2)
    return [
        ("pyramid_clipped", O.make_config(**PYRAMID), 3, _train_config(threshold=1e-3)),
        # unclipped, a step moves ls2 by scale * its gradient (about 1024 coef / N): a small scale keeps sigma near
        # init_sigma, where the cost at step 2 is not dominated by the noise
        ("pyramid_unclipped", O.make_config(**PYRAMID), 3,
         _train_config(threshold=1e8, rules=("momentum",), max_norm=0.0, scale=1e-5)),
        ("timit_content", CO.make_config(**timit), 2, _train_config()),
        ("pyramid_batch1", O.make_config(**PYRAMID), 1, _train_config()),
    ]


@pytest.mark.parametrize("name,cfg,B,tc", _cases(), ids=[c[0] for c in _cases()])
def test_two_steps_match_the_oracle(name, cfg, B, tc):
    """process_batch twice == the oracle's two updates on the replayed eps: the means and ls2 within 1e-4 of each
    parameter's largest entry, the task cost 1e-4, model cost and priors 1e-5 relative, the union's gradient norm."""
    _torch()
    init = CO.init_params if cfg.get("attention_type") == "content" else O.init_params
    params = init(cfg, seed=5, scale=10.0)
    rec = make_recognizer(cfg, params)
    algo = _algorithm(rec, tc)
    ref = {k: np.asarray(v, np.float32).astype(np.float64) for k, v in params.items()}
    ls2 = AN.init_ls2(ref, 1e-2)
    got_ls2 = algo.noise_parameter_values()
    for k, v in ls2.items():
        assert np.array_equal(got_ls2[AN.noise_name(k)], v), k
    state = {}
    for step in range(2):
        batch = O.synthetic_batch(cfg, B=B, T=32, seed=100 + step)
        _, eps = _replay(algo, step)
        ref, ls2, cost, (lc, u, ps2), norm = AN.train_step(cfg, ref, ls2, state, batch, tc, eps, N_EXAMPLES, COEF)
        algo.process_batch(dict(zip(algo.SOURCES, batch)))
        assert abs(float(algo.last_cost.item()) - cost) <= 1e-4 * abs(cost), (step, algo.last_cost.item(), cost)
        st = algo.noise_stats()
        assert abs(st["model_cost"] - lc) <= 1e-5 * abs(lc), (step, st, lc)
        assert abs(st["model_prior_variance"] - ps2) <= 1e-5 * ps2, (step, st, ps2)
        assert abs(st["model_prior_mean"] - u) <= 1e-5 * abs(u) + 1e-9, (step, st, u)
        assert abs(algo.total_gradient_norm() - norm) <= 1e-4 * norm, (step, algo.total_gradient_norm(), norm)
        thr = tc["gradient_threshold"]
        if name.startswith("pyramid_clipped"):
            assert norm > 100 * thr, (step, norm, thr)
        elif name.startswith("pyramid_unclipped"):
            assert norm < thr / 100, (step, norm, thr)
        got = rec.get_parameter_values()
        got_ls2 = algo.noise_parameter_values()
        for k, v in ref.items():
            assert np.abs(got[k] - v).max() <= 1e-4 * np.abs(v).max(), (step, k, np.abs(got[k] - v).max())
            w = ls2[k]
            assert np.abs(got_ls2[AN.noise_name(k)] - w).max() <= 1e-4 * np.abs(w).max(), (step, k)


def test_inference_sees_the_means_and_the_same_seed_gives_the_same_parameters():
    _torch()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    batches = [O.synthetic_batch(cfg, B=3, T=32, seed=100 + s) for s in range(2)]

    def run(seed):
        rec = make_recognizer(cfg, params)
        algo = _algorithm(rec, _train_config(), seed=seed)
        for b in batches:
            algo.process_batch(dict(zip(algo.SOURCES, b)))
        return rec, algo

    rec, algo = run(7)
    x, m, labels, lm = O.synthetic_batch(cfg, B=3, T=32, seed=5)
    means = rec.get_parameter_values()
    fresh = make_recognizer(cfg, means)
    assert np.array_equal(rec.cost(x, m, labels, lm), fresh.cost(x, m, labels, lm))
    # a training forward between updates leaves the means and their packed weights in place for inference
    algo.cost_and_gradients(dict(zip(algo.SOURCES, batches[0])))
    assert np.array_equal(rec.cost(x, m, labels, lm), fresh.cost(x, m, labels, lm))
    same = run(7)[0].get_parameter_values()
    other = run(8)[0].get_parameter_values()
    assert all(np.array_equal(same[k], v) for k, v in means.items())
    assert any(not np.array_equal(other[k], v) for k, v in means.items())


def test_noise_profile_class_runs_only_with_the_noise_on():
    _torch()
    pkg = package()
    lib = pkg._lib.load()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    batch = dict(zip(pkg.GradientDescent.SOURCES, O.synthetic_batch(cfg, B=2, T=24, seed=3)))
    tc = _train_config()
    ms, count = C.c_double(), C.c_int64()

    def launches(algo):
        lib.lvsr_profile_read(b"noise", C.byref(ms), C.byref(count))
        algo.process_batch(batch)
        pkg._lib.check(lib.lvsr_profile_read(b"noise", C.byref(ms), C.byref(count)))
        return count.value

    lib.lvsr_profile_enable(1)
    try:
        off = pkg.GradientDescent(recognizer=make_recognizer(cfg, params),
                                  step_rule=pkg.step_rule_from_config(tc, dict(max_norm=1.0)))
        assert launches(off) == 0
        assert launches(_algorithm(make_recognizer(cfg, params), tc)) > 0
    finally:
        lib.lvsr_profile_enable(0)


STAGES_YAML = """
parent: {base}
training:
    num_batches: 2
stages:
    pretraining:
        number: 0
    main:
        number: 1
        data:
            batch_size: 1
        regularization:
            max_norm: 0
            adaptive_noise:
                model_cost_coefficient: 0.1
                init_sigma: 1.0e-3
    annealing:
        number: 2
        regularization:
            max_norm: 0
            adaptive_noise:
                model_cost_coefficient: 0.1
                init_sigma: 1.0e-3
        training:
            scale: 0.1
"""


def test_compat_three_stages_save_load_and_search(tmp_path, monkeypatch, caplog):
    _torch()
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as LC
    import lvsr.main as M
    pkg = package()
    exp = write_experiment(tmp_path)
    path = os.path.join(str(tmp_path), "stages.yaml")
    with open(path, "w") as f:
        f.write(STAGES_YAML.format(base=exp["base"]))
    cfg = LC.Configuration(path, "$LVSR/lvsr/configs/schema.yaml", [])
    loaded = []
    orig = pkg.GradientDescent.set_noise_parameter_values

    def record(self, values):
        loaded.append({k: np.array(v) for k, v in values.items()})
        return orig(self, values)

    monkeypatch.setattr(pkg.GradientDescent, "set_noise_parameter_values", record)
    out = os.path.join(str(tmp_path), "run")
    with caplog.at_level(logging.INFO):
        M.train_multistage(cfg, out, "", None, None)
    assert "model_prior_variance" in caplog.text and "missing values for parameters" in caplog.text

    def tar_values(name):
        with tarfile.open(os.path.join(out, name)) as tar:
            data = np.load(io.BytesIO(tar.extractfile("_parameters").read()))
            return {k.replace("|", "/"): data[k] for k in data.files}

    main, ann = tar_values("main.tar"), tar_values("annealing.tar")
    noise_keys = sorted(k for k in main if k.startswith("/adaptive_noise."))
    assert "/adaptive_noise.recognizer/encoder/bidir0/forward/fork/fork_inputs.W" in noise_keys
    assert len(noise_keys) == len(main) // 2
    assert not any(k.startswith("/adaptive_noise.") for k in tar_values("pretraining.tar"))
    assert loaded[0] == {} and sorted(loaded[1]) == noise_keys
    assert all(np.array_equal(loaded[1][k], main[k]) for k in noise_keys)
    assert any(not np.array_equal(ann[k], main[k]) for k in noise_keys)          # annealing trained them further
    report = os.path.join(str(tmp_path), "report")
    M.search(cfg.ordered_stages["annealing"], None, os.path.join(out, "annealing.tar"), "valid", "[0]", report, None,
             False, 1)
    with open(os.path.join(report, "report.txt")) as f:
        text = f.read()
    assert "Recognized:" in text and "CER:" in text


@pytest.mark.parametrize("backend", ["nccl", "gloo"])
def test_two_ranks_equal_one_gpu_on_the_concatenated_batch(backend):
    """tests/dist_noise_worker.py under torchrun: two ranks, each with its utterance shard, one all-reduce per step;
    means, log-variances and noise statistics equal the one-GPU run on the whole batch and are identical on both
    replicas.  NCCL needs two GPUs; gloo runs both ranks on whatever GPUs there are (one is enough)."""
    torch = _torch()
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29300 + os.getpid() % 250 + (0 if backend == "nccl" else 250)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port),
                        os.path.join(root, "tests", "dist_noise_worker.py"), backend],
                       capture_output=True, text=True, timeout=600)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "DIST_NOISE_OK" in r.stdout
