// BeamSearch.search for MANY utterances, the whole loop native (libs/blocks/blocks/search.py:244-399 as modified by
// lvsr: char_discount, round_to_inf, stop_on, ignore_first_eol; driven by lvsr/bricks/recognizer.py:513-533).
//
// The per-step device work is search_expand / search_advance (api.cu): one glimpse per hypothesis, readout,
// per-utterance k-best on the GPU, gather + transition.  This file is the reference's host bookkeeping -- histories,
// the `done` list, the two stopping criteria, the final ranking -- in C++, so a step costs one small H2D, one small
// D2H and one stream synchronisation for ALL utterances instead of a Python loop per utterance.  It is the only
// search loop: a validate_solution_function reaches it as the `validate` callback.
//
// Arithmetic that decides orderings is done the way numpy / Python do it there: cumulative costs are float32
// (numpy.take / vstack of float32 arrays), the ranking key `cost - char_discount * len` is float64, sorting is stable.
#include <algorithm>
#include <cmath>
#include <vector>

#include "model.h"

using namespace lvsr;

struct lvsr_search_result {
  struct Hyp { std::vector<int64_t> tokens; std::vector<float> costs; };     // full histories incl. the initial symbol
  std::vector<std::vector<Hyp>> done;                                         // per utterance, ranked
};

namespace {

struct Pinned {
  void* p = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes) {
    if (bytes <= cap) return 0;
    if (p) cudaFreeHost(p);
    p = nullptr; cap = 0;
    LVSR_CUDA_OK(cudaMallocHost(&p, bytes));
    cap = bytes;
    return 0;
  }
  ~Pinned() { if (p) cudaFreeHost(p); }
};

struct Utt {
  std::vector<std::vector<int64_t>> outs;     // live hypotheses: token history (with the initial symbol)
  std::vector<std::vector<float>> costs;      // cumulative cost history (float32 like the reference's arrays)
  std::vector<lvsr_search_result::Hyp> done;
  double min_cost = 1000.0;
  long long patience = 0;
  bool patience_set = false;
  int max_length = 0;
  bool active = true;
};

double discounted(const lvsr_search_result::Hyp& h, double char_discount) {
  return (double)h.costs.back() - char_discount * (double)h.costs.size();      // item[1][-1] - char_discount * len(item[1])
}

}  // namespace

extern "C" {

int lvsr_beam_search_many(lvsr_model* m, const float* attended, const float* preprocessed, const float* attended_mask,
                          int32_t Tp, int32_t U, const int32_t* utt_len_host, const int32_t* max_length_host,
                          int32_t beam_size, int32_t eol_symbol, int32_t ignore_first_eol, double char_discount,
                          double round_to_inf, int32_t stop_on_optimistic, lvsr_validate_fn validate, void* validate_user,
                          lvsr_search_result** result, void* stream) {
  DeviceGuard device_guard(m);
  if (int rc = bind_stream(m, static_cast<cudaStream_t>(stream))) return rc;
  if (int rc = check_ready(m)) return rc;
  LVSR_CHECK(attended && preprocessed && attended_mask && utt_len_host && max_length_host && result && Tp > 0 && U > 0 && beam_size > 0,
             "beam_search_many: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const lvsr_config& c = m->cfg;
  const int C = state_dim(m), E = m->E, V = c.num_phonemes, k = beam_size;     // C: floats of a state row
  const int Rmax = U * k;

  // ---- device state: two sets of (states, weights, step) + the per-step outputs, one allocation -----------------
  auto rnd = [](size_t b) { return (b + 255) & ~(size_t)255; };
  const size_t sz_s = rnd((size_t)Rmax * C * sizeof(float)), sz_w = rnd((size_t)Rmax * Tp * sizeof(float));
  const size_t sz_i64 = rnd((size_t)Rmax * sizeof(long long)), sz_e = rnd((size_t)Rmax * E * sizeof(float));
  const size_t sz_meta = rnd(((size_t)8 * Rmax + 4 * U + 64) * sizeof(int)), sz_cost = rnd((size_t)Rmax * sizeof(float));
  const size_t sz_top = rnd(((size_t)3 * U * k + U) * sizeof(int));
  const size_t total = 3 * sz_s + 6 * sz_w + 4 * sz_i64 + 2 * sz_e + sz_meta + sz_cost + sz_top;
  char* dev = nullptr;
  LVSR_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&dev), total, st));
  struct Free { char* p; cudaStream_t s; ~Free() { if (p) cudaFreeAsync(p, s); } } free_dev{dev, st};
  char* cur = dev;
  auto take = [&](size_t bytes) { char* p = cur; cur += bytes; return p; };
  float* states[2]; float* weights[2]; long long* step[2];
  for (int i = 0; i < 2; ++i) {
    states[i] = reinterpret_cast<float*>(take(sz_s));
    weights[i] = reinterpret_cast<float*>(take(sz_w));
    step[i] = reinterpret_cast<long long*>(take(sz_i64));
  }
  float* tmp_s = reinterpret_cast<float*>(take(sz_s));          // advance output before the finished rows are dropped
  float* tmp_w = reinterpret_cast<float*>(take(sz_w));
  long long* tmp_step = reinterpret_cast<long long*>(take(sz_i64));
  float* wavg = reinterpret_cast<float*>(take(sz_e));           // glimpses of the current rows (expand)
  float* new_w = reinterpret_cast<float*>(take(sz_w));
  float* new_e = reinterpret_cast<float*>(take(sz_w));
  float* n_wavg = reinterpret_cast<float*>(take(sz_e));         // glimpses of the selected children (advance; not carried on)
  float* n_e = reinterpret_cast<float*>(take(sz_w));
  int* d_meta = reinterpret_cast<int*>(take(sz_meta));
  long long* d_sym = reinterpret_cast<long long*>(take(sz_i64));
  float* d_cost = reinterpret_cast<float*>(take(sz_cost));
  int* d_top = reinterpret_cast<int*>(take(sz_top));
  LVSR_CHECK((size_t)(cur - dev) <= total, "beam_search_many: workspace accounting");

  static thread_local Pinned pin_in, pin_out, pin_lm;
  if (int rc = pin_in.ensure(((size_t)8 * Rmax + 4 * U + 64) * sizeof(int) + (size_t)Rmax * (sizeof(long long) + sizeof(float)))) return rc;
  if (int rc = pin_out.ensure(((size_t)3 * U * k + U) * sizeof(int))) return rc;
  int* h_meta = static_cast<int*>(pin_in.p);
  long long* h_sym = reinterpret_cast<long long*>(h_meta + (size_t)8 * Rmax + 4 * U + 64);
  float* h_cost = reinterpret_cast<float*>(h_sym + Rmax);
  int* h_top = static_cast<int*>(pin_out.p);

  // language model state of every row (FSTTransition's states / weights / add), in both sets and the advance scratch
  const bool lm = lm_attached(m);
  int* lm_s[3] = {nullptr, nullptr, nullptr};
  double* lm_w[3] = {nullptr, nullptr, nullptr};
  float* lm_a[3] = {nullptr, nullptr, nullptr};
  unsigned* h_lm = nullptr;
  char* lm_dev = nullptr;
  if (lm) {
    const size_t sz_ls = rnd((size_t)Rmax * LVSR_LM_MAX_STATES * sizeof(int));
    const size_t sz_lw = rnd((size_t)Rmax * LVSR_LM_MAX_STATES * sizeof(double)), sz_la = rnd((size_t)Rmax * V * sizeof(float));
    LVSR_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&lm_dev), 3 * (sz_ls + sz_lw + sz_la), st));
    char* p = lm_dev;
    for (int i = 0; i < 3; ++i) {
      lm_w[i] = reinterpret_cast<double*>(p); p += sz_lw;
      lm_s[i] = reinterpret_cast<int*>(p); p += sz_ls;
      lm_a[i] = reinterpret_cast<float*>(p); p += sz_la;
    }
    if (int rc = pin_lm.ensure(sizeof(unsigned))) return rc;
    h_lm = static_cast<unsigned*>(pin_lm.p);
  }
  struct FreeLm { char* p; cudaStream_t s; ~FreeLm() { if (p) cudaFreeAsync(p, s); } } free_lm{lm_dev, st};
  // the LM status word travels with the step's own copies and is checked after its synchronisations
  auto lm_fetch = [&]() -> int {
    if (lm) LVSR_CUDA_OK(cudaMemcpyAsync(h_lm, m->lm_status.get(), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    return 0;
  };
  auto lm_check = [&]() -> int {
    if (!lm || *h_lm == 0) return 0;
    const unsigned s = *h_lm;
    LVSR_CUDA_OK(cudaMemsetAsync(m->lm_status.get(), 0, sizeof(unsigned), st));
    return lm_report(s);
  };

  // initial states: one row per utterance (B/search.py:103-104: initial_states(1))
  int curset = 0;
  if (int rc = lvsr_initial_states(m, Tp, U, states[0], reinterpret_cast<int64_t*>(tmp_step), wavg, weights[0], new_e,
                                   reinterpret_cast<int64_t*>(step[0]), stream)) return rc;
  if (lm)
    if (int rc = lm_step(lm_fst(m), U, nullptr, nullptr, nullptr, nullptr, lm_s[0], lm_w[0], lm_a[0], st)) return rc;

  std::vector<Utt> utts(U);
  int longest = 0;
  for (int u = 0; u < U; ++u) {
    utts[u].outs.assign(1, std::vector<int64_t>(1, (int64_t)initial_output(m)));   // the emitter's initial output
    utts[u].costs.assign(1, std::vector<float>(1, 0.f));
    utts[u].max_length = max_length_host[u];
    longest = std::max(longest, utts[u].max_length);
  }
  std::vector<int> order(U);
  for (int u = 0; u < U; ++u) order[u] = u;
  auto rank_less = [&](const lvsr_search_result::Hyp& a, const lvsr_search_result::Hyp& b) {
    return discounted(a, char_discount) < discounted(b, char_discount);
  };

  std::vector<int> keep_rows, new_order, widths, sel_widths, keep_after;
  for (int i = 0; i < longest; ++i) {
    // ---- top of the reference loop, per utterance: length limit, empty beam, stopping criterion (:306-332) ----
    keep_rows.clear(); new_order.clear();
    int row0 = 0;
    for (int u : order) {
      Utt& ut = utts[u];
      const int width = (int)ut.outs.size();
      bool stop = i >= ut.max_length || width == 0;
      if (!stop && !stop_on_optimistic) {
        std::stable_sort(ut.done.begin(), ut.done.end(), rank_less);
        if ((int)ut.done.size() > k) ut.done.resize(k);
        if (!ut.done.empty()) {
          const double best = discounted(ut.done[0], char_discount);
          if (best < ut.min_cost) { ut.min_cost = best; ut.patience = 30; ut.patience_set = true; }
          else { ut.patience -= 1; stop = ut.patience == 0; }
        }
      } else if (!stop && stop_on_optimistic) {
        if ((int)ut.done.size() >= k) {
          float mn = INFINITY;
          for (auto& cs : ut.costs) mn = std::min(mn, cs.back());
          const double optimistic = (double)mn - char_discount * (double)ut.max_length;
          const lvsr_search_result::Hyp& last = ut.done[k - 1];                 // `done` is append-ordered here (SURVEY quirk 7)
          stop = ((double)last.costs.back() - char_discount * (double)last.costs.size()) < optimistic;
        }
      }
      if (stop) ut.active = false;
      else {
        new_order.push_back(u);
        for (int r = 0; r < width; ++r) keep_rows.push_back(row0 + r);
      }
      row0 += width;
    }
    if ((int)keep_rows.size() != row0) {
      if (keep_rows.empty()) break;
      const int Rn = (int)keep_rows.size();
      std::copy(keep_rows.begin(), keep_rows.end(), h_meta);
      LVSR_CUDA_OK(cudaMemcpyAsync(d_meta, h_meta, (size_t)Rn * sizeof(int), cudaMemcpyHostToDevice, st));
      const int o = curset ^ 1;
      if (int rc = gather_rows(states[o], states[curset], d_meta, Rn, C, st)) return rc;
      if (int rc = gather_rows(weights[o], weights[curset], d_meta, Rn, Tp, st)) return rc;
      if (int rc = gather_i64(step[o], step[curset], d_meta, Rn, 0, st)) return rc;
      if (lm)
        if (int rc = lm_gather(lm_s[o], lm_w[o], lm_a[o], lm_s[curset], lm_w[curset], lm_a[curset], d_meta, Rn, V, st))
          return rc;
      LVSR_CUDA_OK(cudaStreamSynchronize(st));           // h_meta is reused below
      curset = o;
    }
    order = new_order;
    if (order.empty()) break;

    // ---- one expand for every live hypothesis of every utterance ----
    const int nseg = (int)order.size();
    widths.assign(nseg, 0);
    int R = 0;
    for (int s = 0; s < nseg; ++s) { widths[s] = (int)utts[order[s]].outs.size(); R += widths[s]; }
    int* seg_start = h_meta;                  // [nseg + 1]
    int* row_seg = seg_start + nseg + 1;      // [R]
    int* row_utt = row_seg + R;               // [R]
    int* seg_len = row_utt + R;               // [nseg]
    seg_start[0] = 0;
    for (int s = 0, r = 0; s < nseg; ++s) {
      seg_start[s + 1] = seg_start[s] + widths[s];
      seg_len[s] = utt_len_host[order[s]];
      for (int q = 0; q < widths[s]; ++q, ++r) {
        row_seg[r] = s; row_utt[r] = order[s];
        h_cost[r] = utts[order[s]].costs[q].back();
      }
    }
    const size_t meta_ints = (size_t)nseg + 1 + 2 * R + nseg;
    LVSR_CUDA_OK(cudaMemcpyAsync(d_meta, h_meta, meta_ints * sizeof(int), cudaMemcpyHostToDevice, st));
    LVSR_CUDA_OK(cudaMemcpyAsync(d_cost, h_cost, (size_t)R * sizeof(float), cudaMemcpyHostToDevice, st));
    int* d_seg = d_meta; int* d_rseg = d_seg + nseg + 1; int* d_rutt = d_rseg + R; int* d_len = d_rutt + R;
    int* tp = d_top; int* ts = tp + nseg * k; float* tc = reinterpret_cast<float*>(ts + nseg * k); int* tn = ts + 2 * nseg * k;
    if (int rc = search_expand(m, attended, preprocessed, attended_mask, Tp, U, d_len, d_rutt, d_rseg, d_seg, nseg, R,
                               states[curset], weights[curset], step[curset], d_cost, lm ? lm_a[curset] : nullptr, k, wavg,
                               new_w, new_e, tp, ts, tc, tn, st)) return rc;
    LVSR_CUDA_OK(cudaMemcpyAsync(h_top, d_top, ((size_t)3 * nseg * k + nseg) * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (int rc = lm_fetch()) return rc;
    LVSR_CUDA_OK(cudaStreamSynchronize(st));                 // the step's only synchronisation
    if (int rc = lm_check()) return rc;
    const int* hp = h_top; const int* hs = hp + nseg * k;
    const float* hc = reinterpret_cast<const float*>(hs + nseg * k); const int* hn = hs + 2 * nseg * k;

    // ---- the reference's bookkeeping per utterance (:341-377) ----
    sel_widths.assign(nseg, 0);
    keep_after.clear();
    int base = 0;
    int* parent2 = h_meta;                                   // [Rs] (meta of the advance call, built in place below)
    std::vector<int> par_all; std::vector<long long> sym_all;
    par_all.reserve((size_t)nseg * k); sym_all.reserve((size_t)nseg * k);
    for (int s = 0; s < nseg; ++s) {
      Utt& ut = utts[order[s]];
      const int cnt = hn[s];
      LVSR_CHECK(cnt >= 0, "beam search: non-finite log-probabilities");      // :340 assert numpy.isfinite(logprobs).all()
      std::vector<std::vector<int64_t>> outs2(cnt);
      std::vector<std::vector<float>> costs2(cnt);
      for (int j = 0; j < cnt; ++j) {
        const int p = hp[s * k + j] - seg_start[s];
        outs2[j] = ut.outs[p]; outs2[j].push_back((int64_t)hs[s * k + j]);
        costs2[j] = ut.costs[p]; costs2[j].push_back(hc[s * k + j]);
        par_all.push_back(hp[s * k + j]);
        sym_all.push_back((long long)hs[s * k + j]);
      }
      std::vector<std::vector<int64_t>> outs3;
      std::vector<std::vector<float>> costs3;
      for (int j = 0; j < cnt; ++j) {
        const bool is_eol = outs2[j].back() == (int64_t)eol_symbol;
        const size_t n = costs2[j].size();
        // finished: last symbol is eol and the step's own cost stays below round_to_inf (float32 difference, :365-367)
        if (is_eol && (double)(float)(costs2[j][n - 1] - costs2[j][n - 2]) < round_to_inf) {
          // validate_solution_function (:368-370); the step has synchronised, so nothing is in flight on an abort
          const int32_t valid = validate ? validate(validate_user, order[s], outs2[j].data(), (int32_t)n) : 1;
          LVSR_CHECK(valid >= 0, "beam_search_many: the validate callback failed for utterance %d", order[s]);
          if (valid) {
            lvsr_search_result::Hyp h; h.tokens = outs2[j]; h.costs = costs2[j];
            ut.done.push_back(std::move(h));
          }
        }
        const bool alive = !is_eol || (ignore_first_eol && i == 0);
        if (alive) { keep_after.push_back(base + j); outs3.push_back(std::move(outs2[j])); costs3.push_back(std::move(costs2[j])); }
      }
      ut.outs.swap(outs3); ut.costs.swap(costs3);
      sel_widths[s] = cnt;
      base += cnt;
    }
    // ---- next states of every selected child, then drop the finished ones ----
    const int Rs = base;
    if (Rs == 0) continue;
    int* seg2 = parent2 + Rs; int* rseg2 = seg2 + nseg + 1; int* rutt2 = rseg2 + Rs; int* len2 = rutt2 + Rs; int* keep2 = len2 + nseg;
    std::copy(par_all.begin(), par_all.end(), parent2);
    seg2[0] = 0;
    for (int s = 0, r = 0; s < nseg; ++s) {
      seg2[s + 1] = seg2[s] + sel_widths[s];
      len2[s] = utt_len_host[order[s]];
      for (int q = 0; q < sel_widths[s]; ++q, ++r) { rseg2[r] = s; rutt2[r] = order[s]; h_sym[r] = sym_all[r]; }
    }
    const int nkeep = (int)keep_after.size();
    std::copy(keep_after.begin(), keep_after.end(), keep2);
    const size_t meta2_ints = (size_t)3 * Rs + 2 * nseg + 1 + nkeep;
    LVSR_CUDA_OK(cudaMemcpyAsync(d_meta, h_meta, meta2_ints * sizeof(int), cudaMemcpyHostToDevice, st));
    LVSR_CUDA_OK(cudaMemcpyAsync(d_sym, h_sym, (size_t)Rs * sizeof(long long), cudaMemcpyHostToDevice, st));
    int* d_par = d_meta; int* d_seg2 = d_par + Rs; int* d_rseg2 = d_seg2 + nseg + 1; int* d_rutt2 = d_rseg2 + Rs;
    int* d_len2 = d_rutt2 + Rs; int* d_keep = d_len2 + nseg;
    const int o = curset ^ 1;
    const bool all_kept = nkeep == Rs;
    // advance writes into the other set (or, when rows are dropped afterwards, into scratch that is then compacted)
    float* a_states = all_kept ? states[o] : tmp_s;
    float* a_weights = all_kept ? weights[o] : tmp_w;
    if (int rc = search_advance(m, attended, preprocessed, attended_mask, Tp, U, d_len2, Rs, d_par, d_sym, d_rutt2, d_rseg2,
                                d_seg2, nseg, states[curset], weights[curset], step[curset], wavg, new_w, new_e, a_states,
                                n_wavg, a_weights, n_e, all_kept ? step[o] : tmp_step, st)) return rc;
    const int la = all_kept ? o : 2;                       // FSTTransition.apply of the selected children
    if (lm)
      if (int rc = lm_step(lm_fst(m), Rs, lm_s[curset], lm_w[curset], d_par, d_sym, lm_s[la], lm_w[la], lm_a[la], st))
        return rc;
    if (!all_kept && nkeep > 0) {
      if (int rc = gather_rows(states[o], a_states, d_keep, nkeep, C, st)) return rc;
      if (int rc = gather_rows(weights[o], a_weights, d_keep, nkeep, Tp, st)) return rc;
      if (int rc = gather_i64(step[o], tmp_step, d_keep, nkeep, 0, st)) return rc;
      if (lm)
        if (int rc = lm_gather(lm_s[o], lm_w[o], lm_a[o], lm_s[2], lm_w[2], lm_a[2], d_keep, nkeep, V, st)) return rc;
    }
    if (int rc = lm_fetch()) return rc;
    LVSR_CUDA_OK(cudaStreamSynchronize(st));               // pinned staging is rewritten by the next step
    if (int rc = lm_check()) return rc;
    curset = o;
  }

  lvsr_search_result* res = new lvsr_search_result();
  res->done.resize(U);
  for (int u = 0; u < U; ++u) {
    std::stable_sort(utts[u].done.begin(), utts[u].done.end(), rank_less);      // :382
    res->done[u] = std::move(utts[u].done);
  }
  *result = res;
  return 0;
}

int lvsr_search_result_count(const lvsr_search_result* r, int32_t utt) {
  return (r && utt >= 0 && utt < (int)r->done.size()) ? (int)r->done[utt].size() : -1;
}
int lvsr_search_result_length(const lvsr_search_result* r, int32_t utt, int32_t j) {
  if (!r || utt < 0 || utt >= (int)r->done.size() || j < 0 || j >= (int)r->done[utt].size()) return -1;
  return (int)r->done[utt][j].tokens.size();
}
int lvsr_search_result_get(const lvsr_search_result* r, int32_t utt, int32_t j, int64_t* tokens, float* costs) {
  LVSR_CHECK(r && tokens && costs && utt >= 0 && utt < (int)r->done.size() && j >= 0 && j < (int)r->done[utt].size(),
             "search_result_get: bad index");
  const auto& h = r->done[utt][j];
  std::copy(h.tokens.begin(), h.tokens.end(), tokens);
  std::copy(h.costs.begin(), h.costs.end(), costs);
  return 0;
}
int lvsr_search_result_destroy(lvsr_search_result* r) {
  delete r;
  return 0;
}

}  // extern "C"
