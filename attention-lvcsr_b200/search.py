"""Beam search over the CUDA decoder -- mirror of blocks.search.BeamSearch.

Same constructor/driver contract as the reference's (modified) class
(libs/blocks/blocks/search.py:19-407): ``BeamSearch(beam_size, recognizer)``,
``compile()``, ``search(input_values, eol_symbol, max_length, ...)`` returning
``(outputs, costs)``.  The four compiled Theano functions become four C-ABI calls
(lvsr_encoder_forward, lvsr_initial_states, lvsr_logprobs, lvsr_next_states) for the
state functions, and the search loop itself is ``lvsr_beam_search_many``: all hypothesis
state stays on the GPU, the k-best selection (``_smallest``) happens on the GPU, and the
reference's bookkeeping (histories, ``done`` list, stopping criteria, B/search.py:306-377)
runs in C++, calling back into Python only for ``validate_solution_function``.  ``search_many`` decodes MANY
utterances in lock-step with one set of launches per step (rows index their utterance;
the batch-global window cut of take_glimpses is taken per utterance, exactly as if each
were decoded alone).  Differences from the reference that do not change results: the encoded
sequence is NOT replicated per hypothesis, attention.preprocess runs once per utterance
instead of twice per step, and with the expanding prior the glimpse computed for the
log-probabilities is reused for the state update instead of being recomputed.
"""
import numpy as np

from . import _lib


class CandidateNotFoundError(Exception):
    """libs/blocks/blocks/search.py:15-16."""


def _smallest(matrix, k):
    """k smallest entries of a matrix: ((rows, cols), values), increasing
    (libs/blocks/blocks/search.py:220-242; numpy's argpartition/argsort tie order)."""
    flat = matrix.reshape(-1)
    if flat.shape[0] > k:
        keep = np.argpartition(flat, k)[:k]
    else:
        keep = np.arange(flat.shape[0])
    keep = keep[np.argsort(flat[keep])]
    return np.unravel_index(keep, matrix.shape), flat[keep]


class BeamSearch(object):
    def __init__(self, beam_size, recognizer):
        self.beam_size = beam_size
        self.recognizer = recognizer
        self.compiled = False
        self.context_names = ["attended", "attended_mask"]
        self.state_names = ["states", "outputs", "weighted_averages", "weights", "energies", "step"]

    _smallest = staticmethod(_smallest)

    def compile(self):
        """Nothing to compile: the kernels are ahead-of-time sm_90a code."""
        self.recognizer._require_ready()
        self.compiled = True

    # ---- the four device functions ---------------------------------------------
    def compute_contexts(self, recordings):
        """recordings [T, 1, F] (numpy or torch) -> dict(attended, attended_mask, preprocessed)."""
        r = self.recognizer
        att, mask = r.encode(recordings, None)
        return dict(attended=att, attended_mask=mask, preprocessed=r.preprocess(att))

    def compute_initial_states(self, contexts, width=1):
        return self.recognizer._initial_states(contexts["attended"].shape[0], width)

    def compute_logprobs(self, contexts, states):
        return self.recognizer._logprobs(contexts, states)

    def compute_next_states(self, contexts, states, outputs):
        return self.recognizer._next_states(contexts, states, outputs)

    # ---- driver -----------------------------------------------------------------
    def search(self, input_values, eol_symbol, max_length, ignore_first_eol=False, as_arrays=False,
               char_discount=0, round_to_inf=1e9, stop_on="patience", validate_solution_function=None):
        """See the reference docstring (libs/blocks/blocks/search.py:244-288).
        ``input_values``: {'recordings': array [T, 1, F]} (name or any single key)."""
        (recordings,) = list(input_values.values())
        rec = np.asarray(recordings.cpu() if hasattr(recordings, "cpu") else recordings, dtype=np.float32)
        if rec.ndim != 3 or rec.shape[1] != 1:
            raise ValueError("search expects recordings [T, 1, F]")
        res = self.search_many([rec[:, 0, :]], eol_symbol, [max_length], ignore_first_eol=ignore_first_eol,
                               as_arrays=as_arrays, char_discount=char_discount, round_to_inf=round_to_inf,
                               stop_on=stop_on, validate_solution_function=validate_solution_function,
                               input_values=[input_values])
        return res[0]

    def search_many(self, recordings_list, eol_symbol, max_lengths, ignore_first_eol=False, as_arrays=False,
                    char_discount=0, round_to_inf=1e9, stop_on="patience", validate_solution_function=None,
                    input_values=None, raise_on_failure=True):
        """BeamSearch.search (B/search.py:244-399) for a list of utterances [T_u, F] decoded in lock-step.
        Returns one result per utterance (same format as ``search``); an utterance without a finished
        hypothesis raises CandidateNotFoundError (or yields None with raise_on_failure=False)."""
        import ctypes as C
        if stop_on not in ("patience", "optimistic_future_cost"):
            raise ValueError("Unknown stopping criterion {}".format(stop_on))
        if not self.compiled:
            self.compile()
        r = self.recognizer
        lib, h = _lib.load(), r._require_ready()
        k = int(self.beam_size)
        U = len(recordings_list)
        if U == 0:
            return []
        lens = [int(x.shape[0]) for x in recordings_list]
        Tmax, F = max(lens), int(recordings_list[0].shape[1])
        x = np.zeros((Tmax, U, F), dtype=np.float32)
        for u, a in enumerate(recordings_list):
            x[:lens[u], u, :] = np.asarray(a, dtype=np.float32)
        mask = None
        if min(lens) != Tmax:
            mask = (np.arange(Tmax)[:, None] < np.asarray(lens)[None, :]).astype(np.float32)
        # one encoder pass for all utterances; right-padding is exact under the mask (the masked GRU step returns
        # the carried state bit for bit) and every utterance attends over its own encoded length only
        att, attm = r.encode(x, mask)
        P = r.preprocess(att)
        Tp = int(att.shape[0])
        enc_len = np.asarray([r.encoded_length(t) for t in lens], dtype=np.int32)
        maxl = np.asarray([int(m) for m in max_lengths], dtype=np.int32)
        failure = []
        validate = _lib.VALIDATE_FN()                 # NULL: every finished hypothesis is kept
        if validate_solution_function is not None:
            def call(user, u, tokens, length):
                # an exception cannot cross the C loop: keep it, abort the search with -1 and re-raise it below
                try:
                    iv = input_values[u] if input_values is not None else {"recordings": recordings_list[u][:, None, :]}
                    return 1 if validate_solution_function(iv, np.ctypeslib.as_array(tokens, (length,)).copy()) else 0
                except BaseException as e:
                    failure.append(e)
                    return -1
            validate = _lib.VALIDATE_FN(call)         # this reference keeps the callback alive during the call
        res = C.c_void_p()
        rc = lib.lvsr_beam_search_many(
            h, att.data_ptr(), P.data_ptr(), attm.data_ptr(), Tp, U, enc_len.ctypes.data, maxl.ctypes.data, k,
            int(eol_symbol), int(bool(ignore_first_eol)), float(char_discount or 0), float(round_to_inf),
            1 if stop_on == "optimistic_future_cost" else 0, validate, None, C.byref(res), r._stream())
        if failure:
            raise failure[0]
        _lib.check(rc)
        done_lists = []
        try:
            for u in range(U):
                done = []
                for j in range(lib.lvsr_search_result_count(res, u)):
                    n = lib.lvsr_search_result_length(res, u, j)
                    tok = np.empty((n,), dtype=np.int64)
                    cst = np.empty((n,), dtype=np.float32)
                    _lib.check(lib.lvsr_search_result_get(res, u, j, tok.ctypes.data, cst.ctypes.data))
                    done.append((tok, cst))
                done_lists.append(done)
        finally:
            lib.lvsr_search_result_destroy(res)
        return self._format_results(done_lists, as_arrays, raise_on_failure)

    def _format_results(self, done_lists, as_arrays, raise_on_failure):
        """result_to_lists / the array form of B/search.py:384-407 from ranked `done` lists."""
        results = []
        for done in done_lists:
            if not done:
                if raise_on_failure:
                    raise CandidateNotFoundError()
                results.append(None)
                continue
            max_len = max(seq.shape[0] for seq, _ in done)
            all_outputs = np.zeros((max_len, len(done)))
            all_masks = np.zeros((max_len, len(done)))
            all_costs = np.zeros((max_len, len(done)))
            for j, (seq, cost) in enumerate(done):
                all_outputs[:len(seq), j] = seq
                all_masks[:len(seq), j] = 1
                all_costs[:len(cost), j] = cost
                all_costs[len(cost):, j] = cost[-1]
            result = (all_outputs[1:], all_masks[1:], all_costs[1:] - all_costs[:-1])
            results.append(result if as_arrays else self.result_to_lists(result))
        return results

    @staticmethod
    def result_to_lists(result):
        outputs, masks, costs = [a.T for a in result]
        outputs = [[int(t) for t in out[:int(m.sum())]] for out, m in zip(outputs, masks)]
        costs = [float(c) for c in costs.T.sum(axis=0)]
        return outputs, costs
