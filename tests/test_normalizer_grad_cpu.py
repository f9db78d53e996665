"""The gradient oracle (oracle/lvsr_oracle_grad.py) for the logistic and relu energy normalisers
(lvsr/bricks/attention.py:191-213): autograd of the torch mirror agrees with central finite differences of the
NUMPY oracle's cost, as test_oracle_grad.py checks it for softmax.  These gradients are what the GPU training step
of these normalisers is compared with (test_gpu_normalizer_train.py)."""
from collections import OrderedDict

import numpy as np
import pytest

from oracle import lvsr_oracle as O
from oracle import lvsr_oracle_grad as G

TINY = dict(num_features=5, dims_bidir=[4, 4], subsample=[1, 2], dim_dec=6, dim_matcher=8, conv_n=3,
            conv_num_filters=2, num_phonemes=5, post_merge_dims=[6], maxout_pieces=2)
PRIORS = [None, dict(type="window_around_median", before=3, after=4)]
BIAS = "/recognizer/generator/att_trans/conv_att/energy_comp/linear.b"


@pytest.mark.parametrize("prior", PRIORS, ids=["default", "median"])
@pytest.mark.parametrize("normalizer,bias", [("logistic", -0.7), ("relu", 0.5)])
def test_autograd_matches_finite_differences_of_numpy_oracle(prior, normalizer, bias):
    cfg = O.make_config(prior=prior, energy_normalizer=normalizer, **TINY)
    params = O.init_params(cfg, seed=9, weights_std=0.4, initial_state_std=0.2)
    params["/recognizer/generator/readout/post_merge/bias.b"][:] = np.random.RandomState(0).normal(0, 0.1, 6)
    params[BIAS][:] = bias
    x, m, labels, lm = O.synthetic_batch(cfg, B=2, T=14, seed=6, label_div=4)
    out = O.recognizer_cost(cfg, params, x, m, labels, lm, return_all=True)
    e = out["energies"]
    assert np.isfinite(out["costs"]).all()
    if normalizer == "relu":
        # the relu derivative jumps at 0: every energy of a window (the energies outside it are exactly 0) stays
        # further from 0 than the perturbations below move it, and every window holds a positive one
        inside = e != 0
        assert np.abs(e[inside]).min() > 1e-3
        assert (e > 0).any(axis=-1).all()
        assert (e[inside] < 0).any()                 # both sides of the kink are exercised
    _, grads = G.cost_and_grads(cfg, params, x, m, labels, lm)
    assert np.abs(grads[BIAS]).max() > 1e-6         # the energy bias carries a gradient (softmax has no bias)
    rng = np.random.RandomState(1)

    def cost_of(p):
        return O.batch_cost(O.recognizer_cost(cfg, p, x, m, labels, lm))
    eps = 1e-6
    for name, value in params.items():
        d = rng.normal(size=value.shape)
        plus = OrderedDict(params); minus = OrderedDict(params)
        plus[name] = value + eps * d
        minus[name] = value - eps * d
        fd = (cost_of(plus) - cost_of(minus)) / (2 * eps)
        an = float((grads[name] * d).sum())
        assert abs(fd - an) <= 1e-6 * max(1.0, abs(an)) + 2e-8, (name, fd, an)
