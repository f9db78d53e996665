"""torchrun worker: the data-parallel training step under adaptive weight noise == the 1-GPU step on the concatenated batch.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port P \
        tests/dist_noise_worker.py [nccl|gloo]

Every rank builds the same model with the same noise seed, takes its contiguous utterance shard of ONE global batch
and runs two GradientDescent.process_batch calls: each rank draws the same eps (Philox keyed by seed, update counter
and flat index), the one all-reduce sums the task gradients, and the gradient transform forms g^2 from the GLOBAL mean
gradient.  Rank 0 also runs the same two steps on the whole batch with a second, single-GPU model.  Checked: means,
log-variances and noise_stats against that run (1e-5), and identical means and log-variances on every replica.
With `gloo` the ranks may share one GPU (rank r uses device r mod the device count)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import torch
    import torch.distributed as dist
    from helpers import O, PYRAMID, make_recognizer, package
    backend = sys.argv[1] if len(sys.argv) > 1 else "nccl"
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dev = torch.device("cuda", local % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    if backend == "nccl":
        dist.init_process_group("nccl", device_id=dev)
    else:
        dist.init_process_group("gloo")
    pkg = package()
    cfg = O.make_config(**PYRAMID)
    params = O.init_params(cfg, seed=5, scale=10.0)
    tc = dict(gradient_threshold=2.0, rules=("momentum", "adadelta"), scale=0.5, momentum=0.3, decay_rate=0.95,
              epsilon=1e-6)
    noise = dict(num_examples=40, init_sigma=1e-2, model_cost_coefficient=0.5, seed=3)
    Bg = 4 * world

    def make():
        rec = make_recognizer(cfg, params)
        algo = pkg.GradientDescent(recognizer=rec, step_rule=pkg.step_rule_from_config(tc, dict(max_norm=1.0)),
                                   adaptive_noise=noise)
        algo.initialize()
        return rec, algo

    def state(rec, algo):
        out = dict(rec.get_parameter_values())
        out.update(algo.noise_parameter_values())
        return out

    rec, algo = make()
    batches = [O.synthetic_batch(cfg, B=Bg, T=48, seed=40 + s) for s in range(2)]
    for x, m, labels, lm in batches:
        sl = slice(rank * 4, rank * 4 + 4)
        algo.process_batch(dict(recordings=x[:, sl], recordings_mask=m[:, sl], labels=labels[:, sl], labels_mask=lm[:, sl]))
    got = state(rec, algo)
    stats = algo.noise_stats()
    cost_dp = float(algo.last_cost.item())
    ok = True
    if rank == 0:
        # single-GPU reference on the concatenated batch: hide the process group from GradientDescent
        rec1, algo1 = make()
        algo1._world = lambda: (None, 1)
        for x, m, labels, lm in batches:
            algo1.process_batch(dict(recordings=x, recordings_mask=m, labels=labels, labels_mask=lm))
        want = state(rec1, algo1)
        worst = max(float(np.abs(got[k] - v).max() / max(1e-12, np.abs(v).max())) for k, v in want.items())
        stats1 = algo1.noise_stats()
        worst_stats = max(abs(stats[k] - v) / max(1e-30, abs(v)) for k, v in stats1.items())
        cost1 = float(algo1.last_cost.item())
        print("world %d (%s): worst relative difference of means and ls2 after 2 steps %.3e, noise stats %.3e, "
              "cost %.6f vs %.6f" % (world, backend, worst, worst_stats, cost_dp, cost1))
        ok = worst <= 1e-5 and worst_stats <= 1e-5 and abs(cost_dp - cost1) <= 1e-5 * abs(cost1)
    # every replica must hold identical means, log-variances and noise statistics
    flat = torch.cat([torch.as_tensor(np.asarray(got[k], np.float64)).reshape(-1) for k in sorted(got)] +
                     [torch.tensor([stats[k] for k in sorted(stats)], dtype=torch.float64)])
    flat = flat.to(dev) if backend == "nccl" else flat
    ref = flat.clone()
    dist.broadcast(ref, src=0)
    same = bool((ref == flat).all().item())
    flag = torch.tensor([1.0 if (ok and same) else 0.0])
    flag = flag.to(dev) if backend == "nccl" else flag
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    if flag.item() != 1.0:
        print("rank %d: FAILED (ok=%s identical_replicas=%s)" % (rank, ok, same))
        sys.exit(1)
    if rank == 0:
        print("DIST_NOISE_OK")


if __name__ == "__main__":
    main()
