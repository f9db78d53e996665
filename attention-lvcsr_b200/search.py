"""Beam search over the CUDA decoder -- mirror of blocks.search.BeamSearch.

Same constructor/driver contract as the reference's (modified) class
(libs/blocks/blocks/search.py:19-407): ``BeamSearch(beam_size, recognizer)``,
``compile()``, ``search(input_values, eol_symbol, max_length, ...)`` returning
``(outputs, costs)``.  The four compiled Theano functions become four C-ABI calls
(lvsr_encoder_forward, lvsr_initial_states, lvsr_logprobs, lvsr_next_states) for the
state functions, and the search loop itself runs on ``lvsr_search_expand`` /
``lvsr_search_advance``: all hypothesis state stays on the GPU, the k-best selection
(``_smallest``) happens on the GPU, and only k (parent, symbol, cost) triples per utterance
cross to the host each step, where the reference's bookkeeping (histories, ``done`` list,
stopping criteria, B/search.py:306-377) runs unchanged.  ``search_many`` decodes MANY
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
        import torch
        if stop_on not in ("patience", "optimistic_future_cost"):
            raise ValueError("Unknown stopping criterion {}".format(stop_on))
        if not self.compiled:
            self.compile()
        r = self.recognizer
        lib, h = _lib.load(), r._require_ready()
        dev = r.device
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
        if validate_solution_function is None and not getattr(self, "force_python_loop", False):
            done_lists = self._search_many_native(att, P, attm, Tp, U, enc_len, max_lengths, eol_symbol, ignore_first_eol,
                                                  char_discount, round_to_inf, stop_on)
            return self._format_results(done_lists, as_arrays, raise_on_failure)
        reuse = 1 if r.net["prior"].get("type", "expanding") == "expanding" else 0
        st = r._initial_states(Tp, U)
        states, weights, step = st["states"], st["weights"], st["step"]

        utts = []
        for u in range(U):
            utts.append(dict(outputs=np.full((1, 1), r.net["num_phonemes"], dtype=np.int64),   # initial symbol, recognizer.py:286
                             costs=np.zeros((1, 1), dtype=np.float32), done=[], min_cost=1000, patience=None,
                             max_length=int(max_lengths[u]), active=True))
        order = list(range(U))            # utterances that own rows, in row order (one segment each)

        def discounted(item):
            return item[1][-1] - char_discount * len(item[1])

        def i32(a):
            return torch.as_tensor(np.ascontiguousarray(a, dtype=np.int32), device=dev)

        V = r.net["num_phonemes"]
        for i in range(max(int(m) for m in max_lengths) if U else 0):
            # ---- top of the reference loop, per utterance: length limit, empty beam, stopping criterion ----
            keep_rows, new_order, row0 = [], [], 0
            for u in order:
                ut = utts[u]
                width = ut["outputs"].shape[1]
                stop = i >= ut["max_length"] or width == 0
                if not stop and stop_on == "patience":
                    ut["done"] = sorted(ut["done"], key=discounted)[:k]
                    if ut["done"]:
                        best = discounted(ut["done"][0])
                        if best < ut["min_cost"]:
                            ut["min_cost"], ut["patience"] = best, 30
                        else:
                            ut["patience"] -= 1
                            stop = ut["patience"] == 0
                elif not stop and stop_on == "optimistic_future_cost":
                    if len(ut["done"]) >= k:
                        optimistic = ut["costs"][-1, :].min() - char_discount * ut["max_length"]
                        last = ut["done"][k - 1][1]
                        stop = last[-1] - char_discount * len(last) < optimistic
                if stop:
                    ut["active"] = False
                else:
                    new_order.append(u)
                    keep_rows.extend(range(row0, row0 + width))
                row0 += width
            if len(keep_rows) != row0:
                if not keep_rows:
                    break
                sel = torch.as_tensor(np.asarray(keep_rows, dtype=np.int64), device=dev)
                states, weights, step = states.index_select(0, sel), weights.index_select(0, sel), step.index_select(0, sel)
            order = new_order
            if not order:
                break
            # ---- one expand for every live hypothesis of every utterance ----
            widths = [utts[u]["outputs"].shape[1] for u in order]
            nseg, R = len(order), int(sum(widths))
            seg_start = np.concatenate([[0], np.cumsum(widths)]).astype(np.int32)
            row_seg = np.repeat(np.arange(nseg, dtype=np.int32), widths)
            row_utt = np.repeat(np.asarray(order, dtype=np.int32), widths)
            meta = i32(np.concatenate([seg_start, row_seg, row_utt, enc_len[order]]))
            d_seg, d_rseg, d_rutt, d_len = (meta[:nseg + 1], meta[nseg + 1:nseg + 1 + R], meta[nseg + 1 + R:nseg + 1 + 2 * R],
                                            meta[nseg + 1 + 2 * R:])
            cost_so_far = torch.as_tensor(np.concatenate([utts[u]["costs"][-1] for u in order]).astype(np.float32), device=dev)
            wavg = torch.empty((R, r.dim_encoded), dtype=torch.float32, device=dev)
            new_w = torch.empty((R, Tp), dtype=torch.float32, device=dev)
            new_e = torch.empty((R, Tp), dtype=torch.float32, device=dev)
            top = torch.empty((3 * nseg * k + nseg,), dtype=torch.int32, device=dev)     # parent | symbol | cost bits | count
            tp, ts, tcst, tcnt = top[:nseg * k], top[nseg * k:2 * nseg * k], top[2 * nseg * k:3 * nseg * k], top[3 * nseg * k:]
            states, weights, step = states.contiguous(), weights.contiguous(), step.contiguous()
            _lib.check(lib.lvsr_search_expand(
                h, att.data_ptr(), P.data_ptr(), attm.data_ptr(), Tp, U, d_len.data_ptr(), d_rutt.data_ptr(), d_rseg.data_ptr(),
                d_seg.data_ptr(), nseg, R, states.data_ptr(), weights.data_ptr(), step.data_ptr(), cost_so_far.data_ptr(), k,
                wavg.data_ptr(), new_w.data_ptr(), new_e.data_ptr(), tp.data_ptr(), ts.data_ptr(), tcst.data_ptr(),
                tcnt.data_ptr(), r._stream()))
            top_h = top.cpu().numpy()                                   # the step's only device -> host transfer
            parents_all = top_h[:nseg * k].reshape(nseg, k)
            symbols_all = top_h[nseg * k:2 * nseg * k].reshape(nseg, k)
            costs_all = top_h[2 * nseg * k:3 * nseg * k].view(np.float32).reshape(nseg, k)
            counts = top_h[3 * nseg * k:]
            # ---- the reference's bookkeeping per utterance (B/search.py:341-377) ----
            sel_parent, sel_symbol, sel_widths, keep_after = [], [], [], []
            base = 0
            for sg, u in enumerate(order):
                ut = utts[u]
                cnt = int(counts[sg])
                assert cnt >= 0, "non-finite log-probabilities"          # :340 assert numpy.isfinite(logprobs).all()
                parents = parents_all[sg, :cnt].astype(np.int64) - int(seg_start[sg])
                symbols = symbols_all[sg, :cnt].astype(np.int64)
                chosen = costs_all[sg, :cnt]
                ut["outputs"] = np.vstack([np.take(ut["outputs"], parents, axis=1), symbols[None, :]])
                ut["costs"] = np.vstack([np.take(ut["costs"], parents, axis=1), chosen[None, :].astype(np.float32)])
                alive = symbols != eol_symbol
                if ignore_first_eol and i == 0:
                    alive[:] = True
                ended = np.where((ut["outputs"][-1] == eol_symbol) &
                                 (ut["costs"][-1] - ut["costs"][-2] < round_to_inf))[0]
                for idx in ended:
                    iv = input_values[u] if input_values is not None else {"recordings": recordings_list[u][:, None, :]}
                    if validate_solution_function is None or validate_solution_function(iv, ut["outputs"][:, idx]):
                        ut["done"].append((ut["outputs"][:, idx], ut["costs"][:, idx]))
                keep = np.where(alive)[0]
                sel_parent.append(parents_all[sg, :cnt])
                sel_symbol.append(symbols)
                sel_widths.append(cnt)
                keep_after.extend((base + keep).tolist())
                base += cnt
                ut["outputs"] = np.take(ut["outputs"], keep, axis=1)
                ut["costs"] = np.take(ut["costs"], keep, axis=1)
            # ---- next states of every selected child, then drop the finished ones ----
            Rs = int(sum(sel_widths))
            seg2 = np.concatenate([[0], np.cumsum(sel_widths)]).astype(np.int32)
            meta2 = i32(np.concatenate([np.concatenate(sel_parent), seg2, np.repeat(np.arange(nseg, dtype=np.int32), sel_widths),
                                        np.repeat(np.asarray(order, dtype=np.int32), sel_widths)]))
            d_par, d_seg2, d_rseg2, d_rutt2 = meta2[:Rs], meta2[Rs:Rs + nseg + 1], meta2[Rs + nseg + 1:2 * Rs + nseg + 1], meta2[2 * Rs + nseg + 1:]
            d_sym = torch.as_tensor(np.concatenate(sel_symbol).astype(np.int64), device=dev)
            n_states = torch.empty((Rs, states.shape[1]), dtype=torch.float32, device=dev)
            n_wavg = torch.empty((Rs, r.dim_encoded), dtype=torch.float32, device=dev)
            n_w = torch.empty((Rs, Tp), dtype=torch.float32, device=dev)
            n_e = torch.empty((Rs, Tp), dtype=torch.float32, device=dev)
            n_step = torch.empty((Rs,), dtype=torch.int64, device=dev)
            _lib.check(lib.lvsr_search_advance(
                h, att.data_ptr(), P.data_ptr(), attm.data_ptr(), Tp, U, d_len.data_ptr(), Rs, d_par.data_ptr(), d_sym.data_ptr(),
                d_rutt2.data_ptr(), d_rseg2.data_ptr(), d_seg2.data_ptr(), nseg, states.data_ptr(), weights.data_ptr(),
                step.data_ptr(), wavg.data_ptr(), new_w.data_ptr(), new_e.data_ptr(), reuse, n_states.data_ptr(),
                n_wavg.data_ptr(), n_w.data_ptr(), n_e.data_ptr(), n_step.data_ptr(), r._stream()))
            if len(keep_after) != Rs:
                sel = torch.as_tensor(np.asarray(keep_after, dtype=np.int64), device=dev)
                states, weights, step = n_states.index_select(0, sel), n_w.index_select(0, sel), n_step.index_select(0, sel)
            else:
                states, weights, step = n_states, n_w, n_step

        return self._format_results([sorted(utts[u]["done"], key=discounted) for u in range(U)], as_arrays, raise_on_failure)

    def _search_many_native(self, att, P, attm, Tp, U, enc_len, max_lengths, eol_symbol, ignore_first_eol,
                            char_discount, round_to_inf, stop_on):
        """The loop in C++ (lvsr_beam_search_many): per utterance the ranked `done` list of (tokens, costs) histories."""
        import ctypes as C
        r = self.recognizer
        lib, h = _lib.load(), r._require_ready()
        lens = np.ascontiguousarray(enc_len, dtype=np.int32)
        maxl = np.ascontiguousarray([int(m) for m in max_lengths], dtype=np.int32)
        res = C.c_void_p()
        _lib.check(lib.lvsr_beam_search_many(
            h, att.data_ptr(), P.data_ptr(), attm.data_ptr(), Tp, U, lens.ctypes.data, maxl.ctypes.data, int(self.beam_size),
            int(eol_symbol), int(bool(ignore_first_eol)), float(char_discount or 0), float(round_to_inf),
            1 if stop_on == "optimistic_future_cost" else 0, C.byref(res), r._stream()))
        out = []
        try:
            for u in range(U):
                done = []
                for j in range(lib.lvsr_search_result_count(res, u)):
                    n = lib.lvsr_search_result_length(res, u, j)
                    tok = np.empty((n,), dtype=np.int64)
                    cst = np.empty((n,), dtype=np.float32)
                    _lib.check(lib.lvsr_search_result_get(res, u, j, tok.ctypes.data, cst.ctypes.data))
                    done.append((tok, cst))
                out.append(done)
        finally:
            lib.lvsr_search_result_destroy(res)
        return out

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
