"""The training step of the TIMIT iclr_reward model (exp/timit/configs/iclr_reward.yaml) under log-likelihood,
mse_gain with imitative exploration and mse_gain with greedy exploration, on the GPU, the three alternating step by
step in one process.

    python tools/bench_tle_train.py [--steps 10] [--warmup 3]

Prints one JSON line: for the recipe's batch of 8 and for 64 utterances (T = 800 frames, L = 101 labels, V = 63),
the milliseconds of one GradientDescent.cost_and_gradients-equivalent step (lvsr_train_cost_and_grads, or its greedy
form), median and minimum over CUDA events, and "gpu": the card's name, power limit and maximum SM clock, read in the
same run.  Synthetic inputs and parameters from fixed seeds (bench.py's generators); nothing is written anywhere.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

# exp/timit/configs/iclr_reward.yaml: 123 features, 3 x BiGRU(256) without subsampling, dim_dec 256, matcher 512,
# content+conv attention with the logistic normaliser, Maxout(2) [256], 63 phonemes
ICLR = dict(num_features=123, dims_bidir=[256, 256, 256], subsample=[1, 1, 1], dim_dec=256, dim_matcher=512,
            conv_n=100, conv_num_filters=10, num_phonemes=63, post_merge_dims=[256], maxout_pieces=2,
            energy_normalizer="logistic")
KINDS = (("log_likelihood", "imitative"), ("mse_gain", "imitative"), ("mse_gain", "greedy"))


def make(pkg, dev, net, criterion):
    rec = pkg.SpeechRecognizer(
        input_dims={"recordings": net["num_features"]}, input_num_chars={}, eos_label=net["num_phonemes"] - 1,
        num_phonemes=net["num_phonemes"], dim_dec=net["dim_dec"], dims_bidir=net["dims_bidir"],
        subsample=net["subsample"], conv_n=net["conv_n"], conv_num_filters=net["conv_num_filters"],
        dim_matcher=net["dim_matcher"], post_merge_dims=net["post_merge_dims"], post_merge_activation=pkg.Maxout(2),
        energy_normalizer=net["energy_normalizer"], criterion=dict(name=criterion, min_reward=-5.0),
        enc_transition=pkg.GatedRecurrent, dec_transition=pkg.GatedRecurrent, device=dev)
    rec.set_parameter_values(bench.init_values(rec.parameter_shapes()))
    return rec


def time_steps(torch, pkg, recs, W, steps, warmup, seed):
    x, m, labels, lm = bench.synthetic_batch(W["B"], W["T"], W["F"], W["L"], W["V"], seed=seed)
    algos = {}
    for (crit, expl), rec in recs.items():
        algos[(crit, expl)] = pkg.GradientDescent(recognizer=rec, step_rule=pkg.CompositeRule([pkg.RemoveNotFinite(0.0)]),
                                                  exploration=expl)
        algos[(crit, expl)].initialize()
    batch = dict(recordings=x, recordings_mask=m, labels=labels, labels_mask=lm)
    dev = next(iter(recs.values())).device
    for _ in range(warmup):
        for a in algos.values():
            a._forward_backward(batch, None)
    torch.cuda.synchronize(dev)
    ms = {k: [] for k in algos}
    for _ in range(steps):
        for k, a in algos.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            a._forward_backward(batch, None)
            e1.record()
            torch.cuda.synchronize(dev)
            ms[k].append(e0.elapsed_time(e1))
    return {"%s/%s" % k: {"step_ms_median": round(sorted(v)[len(v) // 2], 3), "step_ms_min": round(min(v), 3)}
            for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_tle_train: needs a CUDA device (no CPU measurement)")
    pkg = __import__("__graft_entry__").load_package()
    dev = torch.device("cuda", 0)
    result = {"gpu": bench.gpu_identity(0)}
    recs = {(crit, expl): make(pkg, dev, ICLR, crit) for crit, expl in KINDS}
    for B in (8, 64):
        W = dict(B=B, T=800, F=ICLR["num_features"], L=101, V=ICLR["num_phonemes"])
        result["B=%d" % B] = dict(time_steps(torch, pkg, recs, W, args.steps, args.warmup, 100 + B),
                                  shape="iclr_reward: 123 features, 3 x BiGRU(256), logistic normaliser, V=63, "
                                        "B=%d x T=800, M=512, L=101" % B)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
