"""lvsr.main of the reference over the GPU engine: the entry points bin/run.py dispatches to
(bin/run.py:140-154 -> lvsr/main.py:522-703 train / train_multistage, :705-865 search, :868-884 sample).

Same function names, arguments and printed report lines; the Blocks main loop, extensions, Bokeh plotting and
the Fuel data pipeline are NOT rebuilt (SURVEY.md section 8: out of scope) -- training is a plain loop over padded
batches calling GradientDescent.process_batch, data comes from the flat .npz of lvsr/datasets/npz.py.
"""
from __future__ import print_function

import logging
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


def train(config, save_path, bokeh_name="", params=None, bokeh_server=None, bokeh=False, test_tag=None,
          use_load_ext=False, load_log=False, fast_start=False):
    """lvsr/main.py:522-703 reduced to its computation: batches -> GradientDescent.process_batch, parameters saved
    in Blocks checkpoint format.  Stops after training.num_epochs (default 1) or training.num_batches."""
    data = Data(**config["data"])
    recognizer = create_model(config, data, params)
    train_conf = config["training"]
    reg_conf = config.get("regularization", {})
    adaptive_noise = None
    if reg_conf.get("adaptive_noise"):
        # lvsr/main.py:425-437: every parameter gets trained Gaussian noise; N is the size of the training set
        logger.info("apply adaptive noise")
        adaptive_noise = dict(reg_conf["adaptive_noise"], num_examples=data.get_dataset("train").num_examples)
    algorithm = pkg.GradientDescent(recognizer=recognizer,
                                    step_rule=pkg.step_rule_from_config(train_conf, reg_conf),
                                    decay=reg_conf.get("decay", 0.0), adaptive_noise=adaptive_noise)
    algorithm.initialize()
    if adaptive_noise and params:
        _load_noise_parameters(algorithm, params)

    def save(path):
        recognizer.save_params(path, extra=algorithm.noise_parameter_values() if adaptive_noise else None)

    num_batches = train_conf.get("num_batches")
    done = 0
    for epoch in range(int(train_conf.get("num_epochs", 1))):
        for batch in data.batches("train", seed=epoch + 1):
            t0 = time.time()
            algorithm.process_batch(batch)
            cost = float(algorithm.last_cost.item())
            done += 1
            # the quantities lvsr/main.py:340-345,357-372 monitors every batch
            logger.info("batch %d: sequence_total_cost %.6f total_gradient_norm %.6f time_train_this_batch %.4f",
                        done, cost, algorithm.total_gradient_norm(), time.time() - t0)
            if adaptive_noise:
                # lvsr/main.py:456-460
                stats = algorithm.noise_stats()
                logger.info("batch %d: task_cost %.6f model_cost %.6f model_prior_mean %.6g model_prior_variance %.6g",
                            done, cost, stats["model_cost"], stats["model_prior_mean"], stats["model_prior_variance"])
            every = train_conf.get("save_every_n_batches")
            if every and done % every == 0 and save_path:
                save(save_path)
            if num_batches and done >= num_batches:
                break
        if num_batches and done >= num_batches:
            break
    if save_path:
        save(save_path)
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
    """lvsr/main.py:896-922: run the stages of a multi-stage configuration in order, each starting from the
    parameters of the previous one."""
    if not getattr(config, "multi_stage", False):
        return train(config, save_path, bokeh_name, params, **kwargs)
    stages = list(config.ordered_stages.items())
    names = [n for n, _ in stages]
    start = names.index(start_stage) if start_stage else 0
    prev = params
    for name, stage_config in stages[start:]:
        stage_path = "%s/%s.tar" % (save_path, name)
        os.makedirs(save_path, exist_ok=True)
        logger.info("training stage %s", name)
        train(stage_config, stage_path, bokeh_name + name, prev, **kwargs)
        prev = stage_path


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
