"""Generate tests/golden/train_golden.npz: float64 gradient oracle (oracle/lvsr_oracle_grad.py) for a WSJ-architecture
training batch big enough to run the production code paths (island-mode persistent decoder: B = 16; tensor-core backward
GEMMs: T*B = 5120 rows), reduced to a few numbers per parameter:

    cost; for every parameter: sum(g), sum(|g|), max|g|, g . r  (r ~ N(0,1) from RandomState(7), drawn in parameter order)

Inputs are regenerated from seeds by the test.  Run from the repo root: python tests/golden/make_train_golden.py (~ minutes)."""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import lvsr_oracle as O  # noqa: E402
from oracle import lvsr_oracle_grad as G  # noqa: E402

WSJ = dict(num_features=40, dims_bidir=[256, 256, 256, 256], subsample=[1, 1, 2, 2], dim_dec=256, dim_matcher=512,
           conv_n=100, conv_num_filters=10, num_phonemes=32, post_merge_dims=[256], maxout_pieces=2)
CASE = dict(B=16, T=320, seed=17)


def reduce_grads(grads, seed=7):
    rng = np.random.RandomState(seed)
    out = {}
    for k, g in grads.items():
        r = rng.normal(size=g.shape)
        out[k] = np.array([g.sum(), np.abs(g).sum(), np.abs(g).max(), (g * r).sum()])
    return out


def main():
    cfg = O.make_config(**WSJ)
    params = O.init_params(cfg, seed=1, scale=10.0)
    batch = O.synthetic_batch(cfg, B=CASE["B"], T=CASE["T"], seed=CASE["seed"])
    t0 = time.time()
    cost, grads = G.cost_and_grads(cfg, params, *batch)
    red = reduce_grads(grads)
    path = os.path.join(ROOT, "tests", "golden", "train_golden.npz")
    np.savez_compressed(path, cost=np.float64(cost), names=np.array(list(red)), stats=np.stack([red[k] for k in red]))
    print("oracle %.1f s, cost %.6f -> %s" % (time.time() - t0, cost, path))


if __name__ == "__main__":
    main()
