"""Task loss estimation on the host: the oracle of tests/tle_oracle.py against the reference's own known answers
(tests/test_error_rate.py of the reference, stored in golden/tle_known_answers.npz) and against a direct restatement
of RewardRegressionEmitter.cost, and the criterion's plumbing through SpeechRecognizer."""
import os
import pickle

import numpy as np
import pytest

import tle_oracle as TO
from helpers import package

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tle_known_answers.npz"))


def _symbols(s):
    return ["abc$".index(c) for c in s]


def test_edit_distance_matrix_known_answer():
    np.testing.assert_array_equal(TO.edit_distance_matrix(*["abdce", "abcd"]), GOLDEN["dist_abdce_abcd"])


@pytest.mark.parametrize("pred", ["abc", "acb"])
def test_reward_and_gain_matrix_known_answers(pred):
    g, y = _symbols("abc$"), _symbols(pred + "$")
    np.testing.assert_array_equal(TO.reward_matrix(g, y, 4, 3), GOLDEN["reward_abc_" + pred])
    np.testing.assert_array_equal(TO.gain_matrix(g, y, 4, 3), GOLDEN["gain_abc_" + pred])


def test_reward_op_is_reward_and_gain_matrix_per_utterance():
    """RewardOp(4, 7) on the reference's test batch: every column is reward_matrix / gain_matrix of the cut sequences,
    padded with -1 / -1000.  (The reference's test_reward_op expects positive rewards, which reward_matrix cannot
    produce since the eos column was added; its inputs are kept, its expected arrays are not.)"""
    g, y = GOLDEN["op_groundtruth"], GOLDEN["op_recognized"]
    rewards, gains = TO.reward_op(g, y, 7, 4)
    for b in range(3):
        gc = list(g[:list(g[:, b]).index(4) + 1, b])
        yc = list(y[:, b])[:list(y[:, b]).index(4) + 1] if 4 in y[:, b] else list(y[:, b])
        n = len(yc)
        np.testing.assert_array_equal(rewards[:n, b], TO.reward_matrix(gc, yc, 7, 4)[:-1])
        np.testing.assert_array_equal(gains[:n, b], TO.gain_matrix(gc, yc, 7, 4)[:-1])
        assert (rewards[n:, b] == -1).all() and (gains[n:, b] == -1000).all()
    rewards, gains = TO.reward_op([[4]], [[1], [2]], 7, 4)                 # lengths differ
    assert rewards.shape == (2, 1, 7)
    with pytest.raises(ValueError, match="EOS"):
        TO.reward_op([[1]], [[1]], 7, 4)


@pytest.mark.parametrize("name", ["mse_gain", "mse_reward"])
@pytest.mark.parametrize("min_reward", [-1.0, -5.0])
def test_tle_cost_equals_a_direct_restatement(name, min_reward):
    """lvsr/bricks/__init__.py:135-184 written out loop by loop."""
    rng = np.random.RandomState(3)
    L, B, V, eos = 7, 3, 6, 5
    y = rng.randint(0, V, size=(L, B))
    y[4, 0] = y[6, 1] = y[2, 2] = eos
    mask = np.zeros((L, B))
    mask[:5, 0] = mask[:, 1] = mask[:3, 2] = 1
    ro = rng.normal(size=(L, B, V))
    R, G = TO.reward_op(y, y, V, eos)
    want = np.zeros((L, B))
    for b in range(B):
        cum = 0.0
        for t in range(L):
            if t > 0:
                cum += ro[t, b, y[t, b]]
            for v in range(V):
                if name == "mse_gain":
                    want[t, b] += (ro[t, b, v] - max(G[t, b, v], min_reward)) ** 2
                else:
                    want[t, b] += (ro[t, b, v] + cum - R[t, b, v]) ** 2
    np.testing.assert_allclose(TO.tle_cost(name, ro, y, R, G, min_reward, mask), want * mask, rtol=1e-12)


def _recognizer(**kw):
    pkg = package()
    return pkg.SpeechRecognizer(input_dims={"recordings": 6}, input_num_chars={}, eos_label=9, num_phonemes=10,
                                dim_dec=64, dims_bidir=[64], conv_n=3, conv_num_filters=4, post_merge_dims=[64],
                                post_merge_activation=pkg.Maxout(2), **kw)


def test_criterion_parsing_and_pickling():
    for name in ("mse_gain", "mse_reward"):
        rec = _recognizer(criterion=dict(name=name, min_reward=-5))
        assert rec.tle and rec.criterion == dict(name=name, min_reward=-5)
        clone = pickle.loads(pickle.dumps(rec))
        assert clone.tle and clone.criterion == rec.criterion
    assert not _recognizer().tle and not _recognizer(criterion=dict(name="log_likelihood")).tle
    with pytest.raises(ValueError, match="Unknown criterion mse_foo"):
        _recognizer(criterion=dict(name="mse_foo"))
    assert package()._lib.CRITERIA == {"log_likelihood": 0, "mse_gain": 1, "mse_reward": 2}


def test_compat_configuration_carries_the_criterion(tmp_path):
    """net.criterion of a recipe (exp/timit/configs/iclr_reward.yaml sets mse_gain, min_reward -5) reaches the
    SpeechRecognizer compat's create_model builds from config['net']."""
    import sys
    from compat_helpers import COMPAT, write_experiment
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as LC
    exp = write_experiment(tmp_path)
    cfg = LC.Configuration(exp["child"], "$LVSR/lvsr/configs/schema.yaml",
                           [("net.criterion", "{name: mse_gain, min_reward: -5}")])
    assert cfg["net"]["criterion"] == dict(name="mse_gain", min_reward=-5)
    net = dict(cfg["net"])
    rec = package().SpeechRecognizer(input_dims={"recordings": 40}, input_num_chars={}, eos_label=11, num_phonemes=12,
                                     **net)
    assert rec.tle and rec.criterion["min_reward"] == -5
