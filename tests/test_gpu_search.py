"""Batched, device-resident beam search (lvsr_beam_search_many, BeamSearch.search_many) against the float64
oracle's line-for-line BeamSearch.search run per utterance: identical token lists, also when a
validate_solution_function filters the finished hypotheses."""
import numpy as np
import pytest

from helpers import O, PYRAMID, make_recognizer, package

pytestmark = pytest.mark.gpu


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _peaky(cfg, seed, gain=10.0, eos_bias=1.0):
    params = O.init_params(cfg, seed=seed, scale=10.0)
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.W"] *= gain
    params["/recognizer/generator/readout/post_merge/mlp/linear_0.b"][cfg["eos_label"]] = eos_bias
    return params


PRIORS = [None, dict(type="window_around_median", before=6, after=8), dict(type="window_around_mean", before=7, after=7),
          dict(type="expanding", initial_begin=0, initial_end=6, min_speed=0.8, max_speed=2.5)]


@pytest.mark.parametrize("prior", PRIORS, ids=lambda p: "default" if p is None else p["type"])
@pytest.mark.parametrize("beam_size,stop_on,char_discount", [(1, "patience", 0), (5, "patience", 0.0),
                                                             (10, "optimistic_future_cost", 0.1)])
def test_search_many_equals_oracle_per_utterance(prior, beam_size, stop_on, char_discount):
    _torch()
    cfg = O.make_config(prior=prior, max_decoded_length_scale=3.0, **PYRAMID)
    params = _peaky(cfg, 11)
    rng = np.random.RandomState(5)
    utts = [rng.normal(size=(T, cfg["num_features"])) for T in (64, 37, 52, 64, 45, 30)]
    rec = make_recognizer(cfg, params)
    rec.init_beam_search(beam_size)
    got = rec._beam_search.search_many([u.astype(np.float32) for u in utts], cfg["eos_label"],
                                       [int(u.shape[0] / 3.0) for u in utts], stop_on=stop_on,
                                       char_discount=char_discount, raise_on_failure=False)
    n_found = n_hyp = 0
    for u, g in zip(utts, got):
        try:
            want = O.beam_search(cfg, params, u, beam_size, stop_on=stop_on, char_discount=char_discount)
        except O.CandidateNotFoundError:
            assert g is None
            continue
        assert g is not None
        n_found += 1
        n_hyp += len(want[0])
        assert g[0] == want[0]
        assert np.allclose(g[1], want[1], rtol=1e-3, atol=5e-3)
    print("utterances with a result:", n_found, "finished hypotheses compared:", n_hyp)
    if beam_size >= 5:
        assert n_found >= 1 and n_hyp >= 3                     # the case is not degenerate
    # the single-utterance entry point is the same code path with one segment
    one = rec.beam_search({"recordings": utts[0]}, stop_on=stop_on, char_discount=char_discount) if got[0] is not None else None
    if one is not None:
        assert one[0] == got[0][0]
    many = rec.beam_search_many([{"recordings": u} for u in utts[:2]], stop_on=stop_on, char_discount=char_discount,
                                raise_on_failure=False)
    assert [None if r is None else r[0] for r in many] == [None if r is None else r[0] for r in got[:2]]


def test_search_launch_count_is_shared_by_all_utterances():
    """Per step ONE expand + ONE advance whatever the number of utterances (the round-1 loop issued two C calls
    of ~6 launches each per utterance and step, and copied the [width, V] table to the host)."""
    _torch()
    pkg = package()
    cfg = O.make_config(max_decoded_length_scale=4.0, **PYRAMID)
    params = _peaky(cfg, 11)
    rng = np.random.RandomState(6)
    utts = [rng.normal(size=(48, cfg["num_features"])).astype(np.float32) for _ in range(12)]
    rec = make_recognizer(cfg, params)
    rec.init_beam_search(4)
    lib = pkg._lib.load()
    lib.lvsr_launch_count(1)
    rec._beam_search.search_many(utts[:1], cfg["eos_label"], [12], raise_on_failure=False)
    one = lib.lvsr_launch_count(1)
    rec._beam_search.search_many(utts, cfg["eos_label"], [12] * 12, raise_on_failure=False)
    many = lib.lvsr_launch_count(1)
    print("launches: 1 utterance", one, "12 utterances", many)
    assert many <= 1.5 * one                              # not 12x


def _validated_case():
    cfg = O.make_config(prior=dict(type="window_around_mean", before=7, after=7), max_decoded_length_scale=2.5, **PYRAMID)
    params = _peaky(cfg, 11, eos_bias=2.0)           # about 50 finished hypotheses, about half of them kept
    rng = np.random.RandomState(8)
    utts = [rng.normal(size=(T, cfg["num_features"])).astype(np.float32) for T in (60, 33, 48, 25, 57)]
    rec = make_recognizer(cfg, params)
    rec.init_beam_search(6)
    return cfg, params, utts, rec, [int(u.shape[0] / 2.5) for u in utts]


def _keep(T, seq):
    """Keeps a finished hypothesis by the parity of its length plus its utterance's frame count, so that a
    validator handed another utterance's inputs decides differently."""
    return (len(seq) + T) % 2 == 0


@pytest.mark.parametrize("stop_on,char_discount", [("patience", 0.0), ("optimistic_future_cost", 0.2)])
def test_validate_solution_function_matches_oracle(stop_on, char_discount):
    """The C++ loop calls validate_solution_function where BeamSearch.search does (B/search.py:365-371): with
    one that rejects some finished hypotheses, every utterance gives the oracle's tokens and costs."""
    _torch()
    cfg, params, utts, rec, maxl = _validated_case()
    ivs = [{"recordings": u[:, None, :]} for u in utts]
    calls = []

    def validate(inputs, seq):
        calls.append((inputs, seq))
        return _keep(inputs["recordings"].shape[0], seq)

    got = rec._beam_search.search_many(utts, cfg["eos_label"], maxl, stop_on=stop_on, char_discount=char_discount,
                                       raise_on_failure=False, validate_solution_function=validate, input_values=ivs)
    n_found = 0
    for u, g in zip(utts, got):
        try:
            want = O.beam_search(cfg, params, u, 6, stop_on=stop_on, char_discount=char_discount,
                                 validate_solution_function=lambda recordings, seq: _keep(recordings.shape[0], seq))
        except O.CandidateNotFoundError:
            assert g is None
            continue
        assert g is not None
        n_found += 1
        assert g[0] == want[0]
        assert np.allclose(g[1], want[1], rtol=1e-3, atol=5e-3)
    kept = [_keep(iv["recordings"].shape[0], seq) for iv, seq in calls]
    print("utterances with a result:", n_found, "validator calls:", len(calls), "kept:", sum(kept))
    assert n_found >= 1 and any(kept) and not all(kept)
    for inputs, seq in calls:
        assert any(inputs is iv for iv in ivs)
        assert seq.dtype == np.int64 and seq[0] == cfg["num_phonemes"] and seq[-1] == cfg["eos_label"]
    # BeamSearch.search hands the validator the caller's own input dict
    u = next(u for u, g in enumerate(got) if g is not None)
    seen = []
    iv = {"recordings": utts[u][:, None, :]}
    rec._beam_search.search(iv, cfg["eos_label"], maxl[u], stop_on=stop_on, char_discount=char_discount,
                            validate_solution_function=lambda inputs, seq: seen.append(inputs) or True)
    assert seen and all(inputs is iv for inputs in seen)


def test_validate_solution_function_rejecting_or_raising():
    """A validator that rejects everything leaves no candidate; an exception it raises reaches the caller as
    itself, and the recognizer searches as before afterwards."""
    _torch()
    cfg, params, utts, rec, maxl = _validated_case()
    bs = rec._beam_search
    before = bs.search_many(utts, cfg["eos_label"], maxl, raise_on_failure=False, as_arrays=True)
    assert any(r is not None for r in before)
    assert bs.search_many(utts, cfg["eos_label"], maxl, raise_on_failure=False,
                          validate_solution_function=lambda inputs, seq: False) == [None] * len(utts)
    with pytest.raises(package().CandidateNotFoundError):
        bs.search_many(utts, cfg["eos_label"], maxl, validate_solution_function=lambda inputs, seq: False)

    def broken(inputs, seq):
        raise ValueError("validator failed on %d tokens" % len(seq))

    with pytest.raises(ValueError, match="validator failed on"):
        bs.search_many(utts, cfg["eos_label"], maxl, validate_solution_function=broken)
    after = bs.search_many(utts, cfg["eos_label"], maxl, raise_on_failure=False, as_arrays=True)
    for a, b in zip(before, after):
        assert (a is None) == (b is None)
        if a is not None:
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
