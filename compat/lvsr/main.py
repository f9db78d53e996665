"""lvsr.main of the reference over the GPU engine: the entry points bin/run.py dispatches to
(bin/run.py:140-154 -> lvsr/main.py:522-703 train / train_multistage, :705-865 search, :868-884 sample).

Same function names, arguments and printed report lines.  Training is a loop over padded batches calling
GradientDescent.process_batch with the extensions of lvsr/main.py that change what is trained, when it stops and
what is saved (validation, PER, best-model checkpoints, Patience, AdaptiveClipping, the NaN stop); Bokeh plotting,
printing filters, pickled main-loop state and the Fuel data pipeline are NOT rebuilt (SURVEY.md section 8: out of
scope) -- data comes from the flat .npz of lvsr/datasets/npz.py.
"""
from __future__ import print_function

import logging
import math
import os
import sys
import time

import numpy

import _engine
from lvsr.datasets import Data

pkg = _engine.pkg
CandidateNotFoundError = pkg.CandidateNotFoundError
logger = logging.getLogger(__name__)


def wer(truth, hyp):
    """Levenshtein distance / len(truth) (lvsr/error_rate.py wer)."""
    d = list(range(len(hyp) + 1))
    for i, t in enumerate(truth, 1):
        prev, d[0] = d[0], i
        for j, h in enumerate(hyp, 1):
            prev, d[j] = d[j], min(d[j] + 1, d[j - 1] + 1, prev + (t != h))
    return d[len(hyp)] / float(max(1, len(truth)))


def create_model(config, data, load_path=None, test_tag=False):
    """lvsr/main.py:206-250: SpeechRecognizer(input dims from the data, **config['net']), the initialisation
    schemes of config['initialization'] set on the bricks their paths name, initialize(), optional parameter load."""
    net = dict(config["net"])
    for unused in ("bottom_class",):
        net.get("bottom", {}).pop(unused, None) if isinstance(net.get("bottom"), dict) else None
    recognizer = pkg.SpeechRecognizer(
        input_dims={"recordings": data.num_features}, input_num_chars={}, eos_label=data.eos_label,
        num_phonemes=data.num_labels, name="recognizer", data_prepend_eos=data.prepend_eos,
        character_map=data.character_map, **net)
    for path, inits in config.get("initialization", {}).items():
        recognizer.set_initialization(path, **inits)
    recognizer.initialize()
    if load_path:
        recognizer.load_params(load_path)
    return recognizer


COST_NAME = "sequence_total_cost"                  # lvsr/main.py:344-345
# AdaptiveClipping as lvsr/main.py:616-619 installs it
CLIPPING_BURNIN_PERIOD, CLIPPING_DECAY_RATE = 500, 0.998


class TrainingLog(object):
    """The part of Blocks' TrainingLog the extensions of lvsr/main.py read: `status` (iterations_done, epochs_done and
    the extensions' entries) and one row of records per iteration."""

    def __init__(self):
        self.status = dict(iterations_done=0, epochs_done=0)
        self.rows = {}

    @property
    def current_row(self):
        return self.rows.setdefault(self.status["iterations_done"], {})


class TrackTheBest(object):
    """blocks.extensions.training.TrackTheBest with choose_best=min: when the current row's `record_name` is lower
    than every earlier value, remember it and write `record_name + "_best_so_far"` = True into the row."""

    def __init__(self, record_name):
        self.record_name = record_name
        self.notification_name = record_name + "_best_so_far"
        self.best_name = "best_" + record_name

    def do(self, log):
        current = log.current_row.get(self.record_name)
        if current is None:
            return
        best = log.status.get(self.best_name)
        if best is None or (current != best and min(current, best) == current):
            log.status[self.best_name] = current
            log.current_row[self.notification_name] = True


class Patience(object):
    """lvsr/extensions.py:157-234 (runs before the first epoch and after every epoch): the last epoch (iteration) whose
    row carries one of `notification_names` is the last best; training stops once
    max(min_epochs, int(patience_factor * last best epoch + 0.5)) <= epochs_done (the iteration variant likewise)."""

    def __init__(self, notification_names, min_iterations=None, min_epochs=None, patience_factor=1.5,
                 patience_log_record=None):
        if (min_epochs is None) == (min_iterations is None):
            raise ValueError("Need exactly one of epochs or iterations to be specified")
        self.notification_names = notification_names
        self.min_iterations, self.min_epochs = min_iterations, min_epochs
        self.patience_factor = patience_factor
        self.last_best_iter = self.last_best_epoch = 0
        self.patience_log_record = patience_log_record or (
            "patience" + ("_epochs" if min_epochs is not None else "_iterations"))

    def do(self, log):
        """Returns True when training should finish."""
        if any(n in log.current_row for n in self.notification_names):
            self.last_best_iter = log.status["iterations_done"]
            self.last_best_epoch = log.status["epochs_done"]
        if self.min_epochs is not None:
            to_do = max(self.min_epochs, int(self.patience_factor * self.last_best_epoch + 0.5))
            done = log.status["epochs_done"]
        else:
            to_do = max(self.min_iterations, int(self.patience_factor * self.last_best_iter + 0.5))
            done = log.status["iterations_done"]
        log.status[self.patience_log_record] = to_do
        return to_do <= done


def _every(n_epochs, n_batches):
    """(after_epoch, after_batch) predicates of set_conditions(every_n_epochs, every_n_batches); 0 / None: never."""
    return (lambda log: bool(n_epochs) and log.status["epochs_done"] % n_epochs == 0,
            lambda log: bool(n_batches) and log.status["iterations_done"] % n_batches == 0)


def validate(recognizer, data):
    """The validation DataStreamMonitoring of lvsr/main.py:550-568,585-592 over `valid` in batches of
    validation_batch_size, unshuffled: the records it adds to the log row."""
    cost = entropy = penalty = labels = utterances = 0.0
    for batch in data.batches("valid", shuffle=False, batch_size=data.validation_batch_size):
        s = recognizer.validation_statistics(batch["recordings"], batch["recordings_mask"], batch["labels"],
                                             batch["labels_mask"])
        cost += s["cost"]
        entropy += s["weights_entropy"]
        penalty += s["weights_penalty"]
        labels += s["num_labels"]
        utterances += s["batch_size"]
    return {"valid_" + COST_NAME: cost / utterances, "valid_num_utterances": utterances,
            "valid_weights_entropy_per_label": entropy / labels,
            "valid_weights_penalty_per_recording": penalty / utterances}


def phoneme_error_rate(recognizer, data, beam_size, char_discount=None, round_to_inf=None, stop_on=None, chunk=None,
                       **unused):
    """PhonemeErrorRate (lvsr/main.py:68-119) over the unbatched `valid` examples, decoded `chunk` utterances at a time
    by beam_search_many.  Its cut-off for hopeless decoding holds in example order: once more than 10 examples are
    scored and their error rate exceeds 0.8, the rate is 1 and no further chunk is decoded."""
    recognizer.init_beam_search(beam_size)
    kwargs = dict(char_discount=char_discount, round_to_inf=round_to_inf, stop_on=stop_on,
                  validate_solution_function=getattr(data.info_dataset, "validate_solution", None))
    kwargs = {k: v for k, v in kwargs.items() if v}
    examples = list(data.examples("valid"))
    chunk = chunk or max(1, data.validation_batch_size)
    total_errors = total_length = 0.0
    num_examples = 0
    for start in range(0, len(examples), chunk):
        group = examples[start:start + chunk]
        results = recognizer.beam_search_many([{"recordings": e["recordings"]} for e in group],
                                              raise_on_failure=False, **kwargs)
        for example, result in zip(group, results):
            if num_examples > 10 and total_errors / total_length > 0.8:
                return 1.0
            groundtruth = data.info_dataset.decode(example["labels"])
            if result is None:                               # CandidateNotFoundError
                error = 1.0
            else:
                error = min(1, wer(groundtruth, data.info_dataset.decode(result[0][0])))
            total_errors += error * len(groundtruth)
            total_length += len(groundtruth)
            num_examples += 1
    return total_errors / total_length


def train(config, save_path, bokeh_name="", params=None, bokeh_server=None, bokeh=False, test_tag=None,
          use_load_ext=False, load_log=False, fast_start=False):
    """lvsr/main.py:522-703 over the GPU engine, with the extensions of initialize_all (:569-675) that change what is
    trained or saved, in their order: validation and PER monitoring, TrackTheBest on both, AdaptiveClipping (on the
    device), FinishAfter(num_batches, num_epochs; default 1 epoch) and the stop on a NaN gradient norm, the `_best` /
    `_best_ll` checkpoints, Patience.  Monitoring runs only when config['monitoring'] has validate_every_* /
    search_every_* keys.  Parameters are saved in Blocks checkpoint format."""
    pkg.algorithms.check_trainable_net(config["net"])     # before the model and the data are built
    train_conf = config["training"]
    reg_conf = config.get("regularization", {})
    # lvsr/main.py:245-283; read under a task-loss criterion only, and refused before any device work
    exploration = pkg.algorithms.check_exploration(
        config["net"], train_conf.get("exploration", "imitative"),
        None if reg_conf.get("adaptive_noise") else {k: reg_conf[k] for k in ("dropout", "noise", "penalty_coof")
                                                     if k in reg_conf})
    data = Data(**config["data"])
    recognizer = create_model(config, data, params)
    mon_conf = config.get("monitoring", {})
    adaptive_noise = None
    if reg_conf.get("adaptive_noise"):
        # lvsr/main.py:425-437: every parameter gets trained Gaussian noise; N is the size of the training set
        logger.info("apply adaptive noise")
        adaptive_noise = dict(reg_conf["adaptive_noise"], num_examples=data.get_dataset("train").num_examples)
    # lvsr/main.py:400-417: dropout on the bottom's output, noise on every parameter outside the attention, the
    # alignment penalty; a config that applies none of them trains exactly as without the keys
    extra = {}
    if reg_conf.get("dropout"):
        logger.info("apply dropout")
    if reg_conf.get("noise"):
        logger.info("apply noise")
    if reg_conf.get("dropout") or reg_conf.get("noise") or reg_conf.get("penalty_coof", 0.0) > 0:
        extra["regularization"] = {k: reg_conf[k] for k in ("dropout", "noise", "penalty_coof") if k in reg_conf}
    if exploration != "imitative":
        extra["exploration"] = exploration
    step_rule = pkg.step_rule_from_config(train_conf, reg_conf)
    if train_conf.get("gradient_threshold"):
        pkg.adaptive_clipping(step_rule, burnin_period=CLIPPING_BURNIN_PERIOD, decay_rate=CLIPPING_DECAY_RATE)
    clipping = pkg.clipping_rule(step_rule)
    algorithm = pkg.GradientDescent(recognizer=recognizer, step_rule=step_rule,
                                    decay=reg_conf.get("decay", 0.0), adaptive_noise=adaptive_noise, **extra)
    algorithm.initialize()
    if adaptive_noise and params:
        _load_noise_parameters(algorithm, params)

    def save(path):
        recognizer.save_params(path, extra=algorithm.noise_parameter_values() if adaptive_noise else None)

    log = TrainingLog()
    validating = "validate_every_epochs" in mon_conf or "validate_every_batches" in mon_conf
    searching = "search_every_epochs" in mon_conf or "search_every_batches" in mon_conf
    valid_epoch, valid_batch = _every(mon_conf.get("validate_every_epochs"), mon_conf.get("validate_every_batches"))
    search_epoch, search_batch = _every(mon_conf.get("search_every_epochs"), mon_conf.get("search_every_batches"))
    track_cost = TrackTheBest("valid_" + COST_NAME)
    track_per = TrackTheBest("valid_per")
    patience = None
    if train_conf.get("patience"):
        patience_conf = dict(train_conf["patience"])
        if not patience_conf.get("notification_names"):
            patience_conf["notification_names"] = [track_per.notification_name, track_cost.notification_name]
        patience = Patience(**patience_conf)
    root, extension = os.path.splitext(save_path) if save_path else (None, None)

    def monitor(on_validation, on_search):
        row = log.current_row
        if validating and on_validation:
            row.update(validate(recognizer, data))
            logger.info("validation after %d batches: %s", log.status["iterations_done"],
                        " ".join("%s %.6g" % kv for kv in sorted(row.items()) if kv[0].startswith("valid_")))
        if searching and on_search:
            row["valid_per"] = phoneme_error_rate(recognizer, data, **mon_conf["search"])
            logger.info("valid_per after %d batches: %.6f", log.status["iterations_done"], row["valid_per"])

    # before_first_epoch
    monitor(not fast_start, not fast_start)
    track_cost.do(log)
    track_per.do(log)
    if patience:
        patience.do(log)
    num_batches = train_conf.get("num_batches")
    num_epochs = int(train_conf.get("num_epochs", 1))
    finish = num_epochs <= 0
    while not finish:
        for batch in data.batches("train", seed=log.status["epochs_done"] + 1):
            t0 = time.time()
            threshold = clipping.current_threshold() if clipping is not None else None
            algorithm.process_batch(batch)
            cost = float(algorithm.last_cost.item())
            log.status["iterations_done"] += 1
            done = log.status["iterations_done"]
            norm = algorithm.total_gradient_norm()
            # the quantities lvsr/main.py:340-345,357-372,542-546 monitors every batch
            logger.info("batch %d: sequence_total_cost %.6f total_gradient_norm %.6f gradient_norm_threshold %.6g "
                        "time_train_this_batch %.4f", done, cost, norm, threshold or 0.0, time.time() - t0)
            if adaptive_noise:
                # lvsr/main.py:456-460
                stats = algorithm.noise_stats()
                logger.info("batch %d: task_cost %.6f model_cost %.6f model_prior_mean %.6g model_prior_variance %.6g",
                            done, cost, stats["model_cost"], stats["model_prior_mean"], stats["model_prior_variance"])
            monitor(valid_batch(log), search_batch(log))
            every = train_conf.get("save_every_n_batches")
            if every and done % every == 0 and save_path:
                save(save_path)
            if math.isnan(norm):
                logger.error("batch %d: the gradient norm is NaN; training stops", done)
                finish = True
            if num_batches and done >= num_batches:
                finish = True
            if finish:
                break
        if finish:
            break
        # after_epoch
        log.status["epochs_done"] += 1
        monitor(valid_epoch(log), search_epoch(log))
        track_cost.do(log)
        track_per.do(log)
        finish = log.status["epochs_done"] >= num_epochs
        if save_path:
            if log.current_row.get(track_per.notification_name):
                save(root + "_best" + extension)
            if log.current_row.get(track_cost.notification_name):
                save(root + "_best_ll" + extension)
        if patience and patience.do(log):
            logger.info("patience: no improvement since epoch %d; training stops after epoch %d",
                        patience.last_best_epoch, log.status["epochs_done"])
            finish = True
    if save_path:
        save(save_path)
    recognizer.training_log = log
    return recognizer


def _load_noise_parameters(algorithm, path):
    """The adaptive-noise parameters of a checkpoint, as Model.set_parameter_values loads them
    (lvsr/main.py:462-470, B/model.py:120-146): the ones present are set, missing ones are logged and keep
    init_sigma (a checkpoint of a stage without adaptive noise has none)."""
    values = algorithm.recognizer.load_checkpoint_values(path)
    want = algorithm.noise_parameter_values()
    found = {k: v for k, v in values.items() if k in want}
    missing = sorted(set(want) - set(found))
    if missing:
        logger.error("missing values for parameters: {}\n".format(missing))
    algorithm.set_noise_parameter_values(found)
    return missing


def train_multistage(config, save_path, bokeh_name, params, start_stage, **kwargs):
    """lvsr/main.py:896-922: run the stages of a multi-stage configuration in order.  The first stage run starts
    from `params`; every later one, and the first when `params` is not given and it is not stage 0, from the
    previous stage's checkpoint <save_path>/<previous stage><training.restart_from>.tar (restart_from "_best_ll":
    the one with the best validation cost)."""
    if not getattr(config, "multi_stage", False):
        return train(config, save_path, bokeh_name, params, **kwargs)
    stages = list(config.ordered_stages.items())
    names = [n for n, _ in stages]
    start = names.index(start_stage) if start_stage else 0
    os.makedirs(save_path, exist_ok=True)
    for number in range(start, len(stages)):
        name, stage_config = stages[number]
        stage_path = "%s/%s.tar" % (save_path, name)
        if number and not params:
            stage_params = "%s/%s%s.tar" % (save_path, names[number - 1],
                                            stage_config["training"].get("restart_from", "") or "")
            if not os.path.exists(stage_params):
                raise IOError("stage %s restarts from %s, which does not exist (restart_from: %r)" % (
                    name, stage_params, stage_config["training"].get("restart_from")))
        else:
            stage_params, params = params, None
        logger.info("training stage %s from %s", name, stage_params or "a fresh initialisation")
        train(stage_config, stage_path, bokeh_name + name, stage_params, **kwargs)


def search(config, params, load_path, part, decode_only, report, decoded_save, nll_only, seed):
    """lvsr/main.py:705-865: groundtruth cost + alignment, beam search, CER per utterance; the printed lines are the
    reference's."""
    data = Data(**config["data"])
    search_conf = config["monitoring"]["search"]
    logger.info("Recognizer initialization started")
    recognizer = create_model(config, data, load_path)
    recognizer.init_beam_search(search_conf["beam_size"])
    logger.info("Recognizer is initialized")
    dataset = data.get_dataset(part)
    if decode_only is not None:
        decode_only = eval(decode_only)
    decoded_file = open(decoded_save, "w") if decoded_save else None
    print_to = sys.stdout
    if report:
        os.makedirs(report, exist_ok=True)
        print_to = open(os.path.join(report, "report.txt"), "w")
    num_examples = total_nll = total_errors = total_length = 0.0
    total_wer_errors = total_word_length = 0.0
    to_words = None
    if config.get("vocabulary"):
        # word error rate over the vocabulary's word ids (lvsr/main.py:757-765)
        with open(os.path.expandvars(config["vocabulary"])) as f:
            vocabulary = dict(line.split() for line in f.readlines())

        def to_words(chars):
            return [vocabulary[w] if w in vocabulary else vocabulary["<UNK>"] for w in chars.split()]
    for number, example in enumerate(data.examples(part, shuffle=part == "train", seed=seed,
                                                   num_examples=500 if part == "train" else None)):
        if decode_only and number not in decode_only:
            continue
        uttids = example.pop("uttids", None)
        raw_groundtruth = example.pop("labels")
        required_inputs = {k: v for k, v in example.items() if k in recognizer.inputs}
        print("Utterance {} ({})".format(number, uttids), file=print_to)
        groundtruth = dataset.decode(raw_groundtruth)
        groundtruth_text = dataset.pretty_print(raw_groundtruth, example)
        costs_groundtruth, weights_groundtruth = recognizer.analyze(
            inputs=required_inputs, groundtruth=raw_groundtruth, prediction=raw_groundtruth)[:2]
        total_nll += costs_groundtruth.sum()
        num_examples += 1
        print("Groundtruth:", groundtruth_text, file=print_to)
        print("Groundtruth cost:", costs_groundtruth.sum(), file=print_to)
        print("Average groundtruth cost: {}".format(total_nll / num_examples), file=print_to)
        if nll_only:
            print_to.flush()
            continue
        before = time.time()
        try:
            search_kwargs = dict(char_discount=search_conf.get("char_discount"),
                                 round_to_inf=search_conf.get("round_to_inf"), stop_on=search_conf.get("stop_on"))
            search_kwargs = {k: v for k, v in search_kwargs.items() if v}
            outputs, search_costs = recognizer.beam_search(required_inputs, **search_kwargs)
        except CandidateNotFoundError:
            logger.error("Candidate not found!")
            outputs = [[]]
            search_costs = [[numpy.nan]]
        took = time.time() - before
        recognized = dataset.decode(outputs[0])
        recognized_text = dataset.pretty_print(outputs[0], example)
        if recognized:
            costs_recognized = recognizer.analyze(inputs=required_inputs, groundtruth=raw_groundtruth,
                                                  prediction=numpy.asarray(outputs[0]))[0]
            error = min(1, wer(groundtruth, recognized))
        else:
            error = 1
        total_errors += len(groundtruth) * error
        total_length += len(groundtruth)
        if to_words:
            wer_error = min(1, wer(to_words(groundtruth_text), to_words(recognized_text)))
            total_wer_errors += len(groundtruth) * wer_error
            total_word_length += len(groundtruth)
        if decoded_file is not None:
            print("{} {}".format(uttids, " ".join(recognized)), file=decoded_file)
        print("Decoding took:", took, file=print_to)
        print("Beam search cost:", search_costs[0], file=print_to)
        print("Recognized:", recognized_text, file=print_to)
        if recognized:
            print("Recognized cost:", costs_recognized.sum(), file=print_to)
        print("CER:", error, file=print_to)
        print("Average CER:", total_errors / total_length, file=print_to)
        if to_words:
            print("WER:", wer_error, file=print_to)
            print("Average WER:", total_wer_errors / total_word_length, file=print_to)
        print_to.flush()
    if decoded_file is not None:
        decoded_file.close()


def sample(config, params, load_path, part):
    """lvsr/main.py:868-884."""
    data = Data(**config["data"])
    recognizer = create_model(config, data, load_path)
    dataset = data.get_dataset(part)
    for number, example in enumerate(data.examples(part)):
        example.pop("uttids", None)
        example.pop("labels")
        print("Utterance", number)
        print(dataset.pretty_print(recognizer.sample(example)[:, 0], example))


def _out_of_scope(name):
    def fn(*args, **kwargs):
        raise NotImplementedError("lvsr.main.%s is outside the GPU hot path (SURVEY.md section 8); "
                                  "available: train_multistage, search, sample" % name)
    fn.__name__ = name
    return fn


test = _out_of_scope("test")
init_norm = _out_of_scope("init_norm")
show_data = _out_of_scope("show_data")
