"""The training loop of lvsr/main.py on the host: the float64 restatements of AdaptiveClipping, Patience, TrackTheBest
and the alignment statistics against hand-worked answers, and compat's main loop (validation, PER, best-model
checkpoints, Patience, the NaN stop, restart_from) with the GPU calls replaced by recording fakes."""
import math
import os
import sys
from collections import OrderedDict

import numpy as np
import pytest

import training_loop_oracle as TL
from compat_helpers import COMPAT, write_experiment
from helpers import package


def test_adaptive_clipping_known_answer():
    # thr0 10, burn-in 2, d 0.5; log norms 1 then 3
    clip = TL.AdaptiveClipping(10.0, 2, 0.5)
    t1 = clip.after_batch(math.e)           # mu .5, mu2 .5, sigma .5, c 1/2
    assert t1 == pytest.approx(0.5 * math.exp(1.0) + 5.0, rel=1e-14)
    t2 = clip.after_batch(math.exp(3.0))    # mu 1.75, mu2 4.75, c 1
    assert t2 == pytest.approx(math.exp(1.75 + math.sqrt(4.75 - 1.75 ** 2)), rel=1e-14)
    assert TL.thresholds_of([math.e, math.exp(3.0), 1.0], 10.0, 2, 0.5) == [10.0, t1, t2]
    # capped at 5 thr0; a zero norm keeps the moments and advances the count; a NaN norm poisons the state
    assert TL.AdaptiveClipping(1.0, 1, 0.0).after_batch(1e6) == 5.0
    z = TL.AdaptiveClipping(10.0, 4, 0.5)
    z.after_batch(math.e)
    mu = z.mean_gradient_norm
    z.after_batch(0.0)
    assert z.mean_gradient_norm == mu and z.iterations_done == 2
    n = TL.AdaptiveClipping(10.0, 4, 0.5)
    n.after_batch(float("nan"))
    assert math.isnan(n.threshold) and math.isnan(n.after_batch(1.0))


def test_track_the_best_and_patience_known_answers():
    assert TL.track_the_best([5.0, None, 4.0, 4.0, 4.5, 3.0]) == [0, 2, 5]
    # last best epoch 2: max(2, int(1.5 * 2 + .5)) = 3
    assert TL.patience_stop_epoch({1, 2}, min_epochs=2, patience_factor=1.5, max_epochs=50) == 3
    assert TL.patience_stop_epoch(set(), min_epochs=4, patience_factor=1.5, max_epochs=50) == 4
    assert TL.patience_stop_epoch({1, 2, 3, 4, 5, 6}, min_epochs=2, patience_factor=1.5, max_epochs=6) is None


def test_alignment_statistics_known_answers():
    w = np.array([[[1.0, 0.0]], [[0.5, 0.5]], [[0.0, 1.0]]])          # L 3, B 1, T' 2
    ent, pen = TL.alignment_stats(w)
    assert ent == pytest.approx(math.log(1 + 1e-7) + 2 * 0.5 * math.log(0.5 + 1e-7) + math.log(1 + 1e-7), rel=1e-14)
    assert pen == 0.0                                                    # the cumsums only move right
    back = np.array([[[0.0, 1.0]], [[1.0, 0.0]]])                       # C0 = [0, 1], C1 = [1, 1]
    assert TL.alignment_stats(back) == (pytest.approx(2 * math.log(1 + 1e-7)), 1.0)
    assert TL.alignment_stats(back, np.array([[1.0], [0.0]]))[1] == 0.0    # step 1 masked: no penalty
    assert TL.alignment_stats(back, np.array([[0.0], [1.0]]))[1] == 1.0    # the mask of step 0 does not enter


LOOP_YAML = """
parent: {base}
data:
    validation_batch_size: 2
training:
    num_epochs: 50
{training}
monitoring:
{monitoring}
"""


def _compat():
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as LC
    import lvsr.main as M
    return LC, M


def _run(tmp_path, monkeypatch, training="", monitoring="    validate_every_epochs: 1\n    search_every_epochs: 1",
         valid_costs=None, pers=None, norms=None, stages=""):
    """compat train_multistage with recording fakes.  valid_costs / pers: the validation cost / PER of each
    validation in order (the first one before the first epoch); norms: gradient norm of each batch."""
    LC, M = _compat()
    pkg = package()
    exp = write_experiment(tmp_path)
    path = os.path.join(str(tmp_path), "loop.yaml")
    with open(path, "w") as f:
        f.write(LOOP_YAML.format(base=exp["base"], training=training, monitoring=monitoring) + stages)
    cfg = LC.Configuration(path, None, [])
    made, calls = [], dict(validations=0, searches=0, batches=0)

    class FakeRecognizer(object):
        lm = None

        def __init__(self, load_path):
            self.load_path = load_path
            self.values = OrderedDict([("/recognizer/generator/readout/post_merge/bias.b", np.zeros(3, np.float32))])

        def get_parameter_values(self):
            return self.values

        save_params = pkg.SpeechRecognizer.save_params
        load_checkpoint_values = staticmethod(pkg.SpeechRecognizer.load_checkpoint_values)

        def validation_statistics(self, x, m, y, ym):
            i = calls["validations"]
            B = x.shape[1]
            return dict(cost=valid_costs[i] * B, weights_entropy=-0.5 * ym.sum(), weights_penalty=0.25 * B,
                        num_labels=float(ym.sum()), batch_size=B)

    class FakeGD(object):
        def __init__(self, recognizer, step_rule, decay, adaptive_noise):
            self.recognizer, self.step_rule = recognizer, step_rule
            made.append(self)

        def initialize(self):
            pass

        def process_batch(self, batch):
            calls["batches"] += 1
            self.last_cost = np.float32(1.5)
            self.recognizer.values["/recognizer/generator/readout/post_merge/bias.b"][:] = calls["batches"]

        def total_gradient_norm(self):
            return 0.5 if norms is None else norms[calls["batches"] - 1]

    real_validate = M.validate

    def validate(recognizer, data):
        out = real_validate(recognizer, data)
        calls["validations"] += 1
        return out

    def per(recognizer, data, **kw):
        calls["searches"] += 1
        return pers[calls["searches"] - 1]

    monkeypatch.setattr(M, "create_model", lambda config, data, load_path=None, test_tag=False: FakeRecognizer(load_path))
    monkeypatch.setattr(M.pkg, "GradientDescent", FakeGD)
    monkeypatch.setattr(M, "validate", validate)
    monkeypatch.setattr(M, "phoneme_error_rate", per)
    out = os.path.join(str(tmp_path), "run")
    if stages:
        M.train_multistage(cfg, out, "", None, None)
    else:
        os.makedirs(out)
        M.train(cfg, os.path.join(out, "loop.tar"))
    return out, made, calls


def _saved_bias(path):
    pkg = package()
    return float(pkg.SpeechRecognizer.load_checkpoint_values(path)["/recognizer/generator/readout/post_merge/bias.b"][0])


def test_patience_stop_epoch_and_best_checkpoints(tmp_path, monkeypatch):
    # 10 training utterances in batches of 4: 3 batches per epoch.  Validation before epoch 1 and after each epoch.
    valid_costs = [5.0, 4.0, 3.0, 3.5, 3.6, 3.7, 3.8, 3.9, 4.0, 4.1]
    pers = [1.0, 0.5, 0.6, 0.7, 0.7, 0.7, 0.7, 0.7, 0.7, 0.7]
    out, made, calls = _run(tmp_path, monkeypatch, training="    patience:\n        min_epochs: 2\n"
                                                            "        patience_factor: 1.5",
                            valid_costs=valid_costs, pers=pers)
    best_cost = [i for i in TL.track_the_best(valid_costs)]              # rows 0 (before epoch 1), 1, 2
    best_per = [i for i in TL.track_the_best(pers)]
    stop = TL.patience_stop_epoch(set(best_cost + best_per) - {0}, 2, 1.5, 50)
    assert stop == 3
    assert calls["batches"] == 3 * stop and calls["validations"] == stop + 1 and calls["searches"] == stop + 1
    assert sorted(os.listdir(out)) == ["loop.tar", "loop_best.tar", "loop_best_ll.tar"]
    assert _saved_bias(os.path.join(out, "loop_best_ll.tar")) == 3 * max(best_cost)     # after epoch 2
    assert _saved_bias(os.path.join(out, "loop_best.tar")) == 3 * max(best_per)         # after epoch 1
    assert _saved_bias(os.path.join(out, "loop.tar")) == 3 * stop
    log = made[0].recognizer.training_log
    assert log.status["epochs_done"] == stop and log.status["patience_epochs"] == 3
    row = log.rows[6]
    assert row["valid_sequence_total_cost"] == pytest.approx(3.0) and row["valid_per"] == pytest.approx(0.6)
    assert row["valid_num_utterances"] == 3 and row["valid_weights_penalty_per_recording"] == pytest.approx(0.25)
    assert row["valid_weights_entropy_per_label"] == pytest.approx(-0.5)
    # the clipping rule the algorithm got is marked adaptive with the reference's constants
    clip = package().clipping_rule(made[0].step_rule)
    assert clip.adaptive == dict(burnin_period=500, decay_rate=0.998) and clip.current_threshold() == 10.0


def test_hopeless_decoding_cut_off_in_example_order(tmp_path):
    LC, M = _compat()
    exp = write_experiment(tmp_path, n_valid=14)
    data = M.Data(path=exp["npz"], batch_size=4)
    seen = []

    class Rec(object):
        def init_beam_search(self, beam_size):
            pass

        def beam_search_many(self, inputs, **kw):
            seen.append(len(inputs))
            return [None for _ in inputs]            # every utterance fails: error 1

    assert M.phoneme_error_rate(Rec(), data, beam_size=2, chunk=4) == 1.0
    assert seen == [4, 4, 4]                         # the 12th example is refused: the fourth chunk is not decoded


def test_nan_gradient_norm_stops_the_loop(tmp_path, monkeypatch):
    out, made, calls = _run(tmp_path, monkeypatch, monitoring="    search:\n        beam_size: 2",
                            norms=[0.5, float("nan"), 0.5, 0.5])
    assert calls["batches"] == 2 and calls["validations"] == 0
    assert sorted(os.listdir(out)) == ["loop.tar"]


def test_config_without_monitoring_keys_trains_as_before(tmp_path, monkeypatch):
    out, made, calls = _run(tmp_path, monkeypatch, training="    num_epochs: 2",
                            monitoring="    search:\n        beam_size: 2")
    assert calls == dict(validations=0, searches=0, batches=6)
    assert sorted(os.listdir(out)) == ["loop.tar"] and _saved_bias(os.path.join(out, "loop.tar")) == 6


STAGES = """
stages:
    pretraining:
        number: 0
        training:
            num_epochs: 3
    main:
        number: 1
        training:
            num_epochs: 1
            restart_from: _best_ll
"""


def test_restart_from_loads_the_best_ll_checkpoint(tmp_path, monkeypatch):
    out, made, calls = _run(tmp_path, monkeypatch, monitoring="    validate_every_epochs: 1",
                            valid_costs=[5.0, 3.0, 4.0, 4.5, 2.0, 1.0], stages=STAGES)
    pre, main = made
    assert pre.recognizer.load_path is None
    assert main.recognizer.load_path == os.path.join(out, "pretraining_best_ll.tar")
    assert _saved_bias(main.recognizer.load_path) == 3.0                 # after epoch 1 of pretraining
    assert "main_best_ll.tar" in os.listdir(out)


def test_restart_from_a_missing_checkpoint_is_an_error(tmp_path, monkeypatch):
    with pytest.raises(IOError, match="pretraining_best_ll.tar"):
        _run(tmp_path, monkeypatch, monitoring="    search:\n        beam_size: 2", stages=STAGES)


def test_adaptive_clipping_marks_the_rule_and_checks_its_arguments():
    pkg = package()
    rule = pkg.step_rule_from_config(dict(gradient_threshold=100.0, scale=0.01, momentum=0.0))
    assert pkg.adaptive_clipping(rule, burnin_period=3, decay_rate=0.9) is rule
    clip = pkg.clipping_rule(rule)
    assert clip.adaptive == dict(burnin_period=3, decay_rate=0.9) and clip.current_threshold() == 100.0
    # the chain maps onto the same train config: the threshold is the initial one
    assert pkg.algorithms._to_train_config(rule).gradient_threshold == 100.0
    with pytest.raises(ValueError):
        pkg.adaptive_clipping(pkg.CompositeRule([pkg.StepClipping(None), pkg.RemoveNotFinite(0.0)]))
    with pytest.raises(ValueError):
        pkg.adaptive_clipping(pkg.CompositeRule([pkg.Momentum(0.1, 0.0), pkg.RemoveNotFinite(0.0)]))
    with pytest.raises(ValueError):
        pkg.adaptive_clipping(rule, burnin_period=0)
