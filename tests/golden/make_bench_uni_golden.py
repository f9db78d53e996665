"""Generate tests/golden/bench_uni_golden.npz: the float64 gradient oracle of the forward-only training step
tools/bench_unidirectional.py times -- bench.NET with bidir False (4 forward GRU layers of 256, encoded width 256),
bench.init_values over its parameter shapes, and the inputs of the first shard of bench.TRAIN_WORKLOAD (64 utterances
of up to 1500 frames, 190 label steps).

Everything but the model is make_bench_train_golden.py's, imported from it: the gradient is the mean of the gradients
of the utterances cropped to their own frames and labels (exact under the default prior: a padded frame leaves the
masked forward state unchanged and a padded label costs 0; tests/test_bench_uni_golden_cpu.py checks this on small
configs), the readout's maxout units near a kink are moved off it by their own bias offsets (kink_nudges, computed
here for this model's readout), and the fixture stores the same digests, statistics and entries.  The oracle is
tests/unidirectional_oracle.py.

Run from the repo root (about 4 minutes on 8 CPU cores):
    python tests/golden/make_bench_uni_golden.py [--workers N] [--out PATH]
"""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
# tests/golden too: the generator's spawned workers import make_bench_train_golden by name to run its worker functions
for p in (ROOT, os.path.join(ROOT, "tests"), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)
import bench  # noqa: E402
import make_bench_train_golden as base  # noqa: E402
import unidirectional_oracle as U  # noqa: E402

PATH = os.path.join(HERE, "bench_uni_golden.npz")
SEED = base.SEED                   # bench.train_bench's inputs on rank 0
ORACLE = "unidirectional_oracle"   # the module the generator's workers import (tests/ is on their path)
NET = dict(bench.NET, bidir=False)


def bench_inputs():
    """(cfg, batch, float32 params) of the forward-only benchmark step; params in U.param_shapes order, as
    tools/bench_unidirectional.py draws them (bench.init_values over the recognizer's parameter shapes)."""
    cfg = U.make_config(**bench.NET)
    params = bench.init_values(U.param_shapes(cfg))
    batch = bench.synthetic_batch(**bench.TRAIN_WORKLOAD, seed=SEED)
    return cfg, batch, params


def meta():
    return dict(workload=bench.TRAIN_WORKLOAD, net=NET, train_conf=bench.TRAIN_CONF, seed=SEED)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workers", type=int, default=min(8, os.cpu_count() or 1))
    ap.add_argument("--out", default=PATH)
    args = ap.parse_args()
    cfg, batch, params = bench_inputs()
    base.write_fixture(args.out, cfg, batch, params, meta(), args.workers, oracle=ORACLE)


if __name__ == "__main__":
    main()
