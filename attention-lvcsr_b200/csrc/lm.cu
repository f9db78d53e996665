// FST language model for shallow fusion (lvsr/ops.py:22-233, lvsr/bricks/language_models.py).
//
// The state of a hypothesis is a set of at most LVSR_LM_MAX_STATES (fst state, weight) pairs, weights being costs
// (negative log).  Advancing by a symbol is transition (every arc with that label, weights log-added per next
// state) followed by the epsilon closure; the cost row of a set is, per symbol, the log-sum of the advanced set minus
// the log-sum of the set itself, or no_transition_cost when the symbol leads nowhere.
//
// All weights and log-adds are float64: a hypothesis accumulates arc weights over hundreds of symbols and a cost is
// a difference of two such sums, so float32 would lose about 1e-3 absolute.  Only the cost row is rounded to float32,
// as the reference stores it.  The arc table is CSR in NN label space (label = symbol + 1, 0 = epsilon), each
// state's arcs sorted by (label, next state), so a state's epsilon arcs come first and a symbol's arcs are found by
// binary search.
//
// Sets over LVSR_LM_MAX_STATES, closures over LM_CLOSURE_CAP states and epsilon cycles (self-loops included) are
// reported in the status word (first error wins); the host turns it into an error return.
#include <math.h>

#include "kernels.h"
#include "lvsr_b200.h"

namespace lvsr {

namespace {

constexpr int LM_CLOSURE_CAP = 32;
constexpr int LM_WARPS = 4;

__device__ __forceinline__ void lm_fail(unsigned* status, unsigned code) { atomicCAS(status, 0u, code); }

// -log(exp(-a) + exp(-b)): the min form of combine_weights, one term at a time (+inf = no term yet)
__device__ __forceinline__ double lm_logadd(double a, double b) {
  if (isinf(a)) return b;
  if (isinf(b)) return a;
  const double lo = fmin(a, b), hi = fmax(a, b);
  return lo - log1p(exp(lo - hi));
}

__device__ __forceinline__ long long lm_first_arc(const LmFst& f, long long lo, long long hi, int label) {
  while (lo < hi) {                      // lower_bound on the label within one state's sorted arcs
    const long long mid = (lo + hi) >> 1;
    if (f.label[mid] < label) lo = mid + 1; else hi = mid;
  }
  return lo;
}

struct LmSet {
  int n;
  int s[LM_CLOSURE_CAP];
  double w[LM_CLOSURE_CAP];
};

__device__ __forceinline__ int lm_find(const LmSet& t, int state) {
  for (int k = 0; k < t.n; ++k)
    if (t.s[k] == state) return k;
  return -1;
}

// expand(transition(src, label)) into out (label < 0: expand(src)).  Returns false on a closure over the cap or an
// epsilon cycle (status set).
__device__ bool lm_advance(const LmFst& f, const int* src_s, const double* src_w, int nsrc, int label, LmSet& out) {
  out.n = 0;
  if (label < 0) {
    for (int i = 0; i < nsrc; ++i) { out.s[out.n] = src_s[i]; out.w[out.n] = src_w[i]; out.n++; }
  } else {
    for (int i = 0; i < nsrc; ++i) {
      const long long end = f.off[src_s[i] + 1];
      for (long long j = lm_first_arc(f, f.off[src_s[i]], end, label); j < end && f.label[j] == label; ++j) {
        const double v = src_w[i] + (double)f.weight[j];
        const int k = lm_find(out, f.next[j]);
        if (k >= 0) { out.w[k] = lm_logadd(out.w[k], v); continue; }
        if (out.n == LM_CLOSURE_CAP) { lm_fail(f.status, LVSR_LM_CLOSURE_CAP); return false; }
        out.s[out.n] = f.next[j]; out.w[out.n] = v; out.n++;
      }
    }
  }
  // epsilon closure: every state reachable over epsilon arcs, in-degree within the closure, then Kahn's order
  unsigned char indeg[LM_CLOSURE_CAP];
  for (int k = 0; k < out.n; ++k) indeg[k] = 0;
  for (int q = 0; q < out.n; ++q) {
    const long long end = f.off[out.s[q] + 1];
    for (long long j = f.off[out.s[q]]; j < end && f.label[j] == 0; ++j) {
      int k = lm_find(out, f.next[j]);
      if (k < 0) {
        if (out.n == LM_CLOSURE_CAP) { lm_fail(f.status, LVSR_LM_CLOSURE_CAP); return false; }
        k = out.n++;
        out.s[k] = f.next[j]; out.w[k] = INFINITY; indeg[k] = 0;
      }
      indeg[k]++;
    }
  }
  unsigned char order[LM_CLOSURE_CAP];
  int head = 0, tail = 0;
  for (int k = 0; k < out.n; ++k)
    if (indeg[k] == 0) order[tail++] = (unsigned char)k;
  while (head < tail) {
    const int k = order[head++];          // every predecessor has been added in: out.w[k] is final
    const long long end = f.off[out.s[k] + 1];
    for (long long j = f.off[out.s[k]]; j < end && f.label[j] == 0; ++j) {
      const int d = lm_find(out, f.next[j]);
      out.w[d] = lm_logadd(out.w[d], out.w[k] + (double)f.weight[j]);
      if (--indeg[d] == 0) order[tail++] = (unsigned char)d;
    }
  }
  if (tail != out.n) { lm_fail(f.status, LVSR_LM_CYCLE); return false; }
  return true;
}

__device__ __forceinline__ double lm_total(const int* s, const double* w, int n) {
  double t = INFINITY;
  for (int i = 0; i < n; ++i) t = lm_logadd(t, w[i]);
  return t;
}

// Per-warp shared copy of the current set.
struct LmShared {
  int n;
  int s[LVSR_LM_MAX_STATES];
  double w[LVSR_LM_MAX_STATES];
};

// Lane 0: sh = expand(transition(sh, label)) (label < 0: expand of sh).  Whole warp afterwards.
__device__ void lm_warp_advance(const LmFst& f, LmShared& sh, int label, int lane) {
  if (lane == 0) {
    LmSet t;
    int n = 0;
    if (lm_advance(f, sh.s, sh.w, sh.n, label, t)) {
      if (t.n > LVSR_LM_MAX_STATES) lm_fail(f.status, LVSR_LM_TOO_MANY_STATES);
      n = min(t.n, (int)LVSR_LM_MAX_STATES);
      for (int i = 0; i < n; ++i) { sh.s[i] = t.s[i]; sh.w[i] = t.w[i]; }
    }
    sh.n = n;
  }
  __syncwarp();
}

// FSTCostsOp row of the set in sh, lanes over the symbols.
__device__ void lm_warp_costs(const LmFst& f, const LmShared& sh, float* add_row, int lane) {
  const double total = lm_total(sh.s, sh.w, sh.n);
  for (int v = lane; v < f.V; v += 32) {
    float cost = f.no_transition_cost;
    if (sh.n > 0) {
      LmSet t;
      if (lm_advance(f, sh.s, sh.w, sh.n, v + 1, t) && t.n > 0)
        cost = (float)(lm_total(t.s, t.w, t.n) - total);
    }
    add_row[v] = cost;
  }
}

__global__ void __launch_bounds__(32 * LM_WARPS) lm_step_kernel(LmFst f, int R, const int* src_states,
                                                                 const double* src_weights, const int* parent,
                                                                 const long long* symbols, int* states_out,
                                                                 double* weights_out, float* add_out) {
  __shared__ LmShared shm[LM_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = blockIdx.x * LM_WARPS + warp;
  if (r >= R) return;
  LmShared& sh = shm[warp];
  if (lane == 0) {
    sh.n = 0;
    if (!symbols) {
      sh.s[0] = f.start; sh.w[0] = 0.0; sh.n = 1;              // expand({start: 0})
    } else {
      const int p = parent ? parent[r] : r;
      for (int i = 0; i < LVSR_LM_MAX_STATES; ++i) {
        const int s = src_states[(long long)p * LVSR_LM_MAX_STATES + i];
        if (s >= 0) { sh.s[sh.n] = s; sh.w[sh.n] = src_weights[(long long)p * LVSR_LM_MAX_STATES + i]; sh.n++; }
      }
    }
  }
  __syncwarp();
  lm_warp_advance(f, sh, symbols ? (int)symbols[r] + 1 : -1, lane);
  if (lane < LVSR_LM_MAX_STATES) {
    states_out[(long long)r * LVSR_LM_MAX_STATES + lane] = lane < sh.n ? sh.s[lane] : -1;   // NOT_STATE padding
    weights_out[(long long)r * LVSR_LM_MAX_STATES + lane] = lane < sh.n ? sh.w[lane] : 0.0;
  }
  lm_warp_costs(f, sh, add_out + (long long)r * f.V, lane);
}

// Teacher forcing (LanguageModel.evaluate): one warp per utterance walks its labels; add[i] is the row in force
// before label i, and a masked label leaves the set as it is.
__global__ void __launch_bounds__(32 * LM_WARPS) lm_path_kernel(LmFst f, int L, int B, const long long* labels,
                                                                 const float* lmask, float* add) {
  __shared__ LmShared shm[LM_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.x * LM_WARPS + warp;
  if (b >= B) return;
  LmShared& sh = shm[warp];
  if (lane == 0) { sh.s[0] = f.start; sh.w[0] = 0.0; sh.n = 1; }
  __syncwarp();
  lm_warp_advance(f, sh, -1, lane);
  for (int i = 0; i < L; ++i) {
    if (i > 0 && (!lmask || lmask[(long long)(i - 1) * B + b] != 0.f))
      lm_warp_advance(f, sh, (int)labels[(long long)(i - 1) * B + b] + 1, lane);
    lm_warp_costs(f, sh, add + ((long long)i * B + b) * f.V, lane);
    __syncwarp();
  }
}

__global__ void lm_gather_kernel(int* states, double* weights, float* add, const int* src_states,
                                 const double* src_weights, const float* src_add, const int* idx, int Rn, int V) {
  const int r = blockIdx.x, t = threadIdx.x;
  const int p = idx[r];
  if (t < LVSR_LM_MAX_STATES) {
    states[(long long)r * LVSR_LM_MAX_STATES + t] = src_states[(long long)p * LVSR_LM_MAX_STATES + t];
    weights[(long long)r * LVSR_LM_MAX_STATES + t] = src_weights[(long long)p * LVSR_LM_MAX_STATES + t];
  }
  for (int v = t; v < V; v += blockDim.x) add[(long long)r * V + v] = src_add[(long long)p * V + v];
}

}  // namespace

int lm_step(const LmFst& f, int R, const int* src_states, const double* src_weights, const int* parent,
            const long long* symbols, int* states_out, double* weights_out, float* add_out, cudaStream_t stream) {
  ProfScope prof("lm", stream);
  if (R <= 0) return 0;
  LVSR_CHECK(f.V >= 1 && f.V <= 128, "lm: num_phonemes %d outside [1, 128]", f.V);
  lm_step_kernel<<<ceil_div(R, LM_WARPS), 32 * LM_WARPS, 0, stream>>>(f, R, src_states, src_weights, parent, symbols,
                                                                       states_out, weights_out, add_out);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int lm_path(const LmFst& f, int L, int B, const long long* labels, const float* lmask, float* add, cudaStream_t stream) {
  ProfScope prof("lm", stream);
  if (L <= 0 || B <= 0) return 0;
  lm_path_kernel<<<ceil_div(B, LM_WARPS), 32 * LM_WARPS, 0, stream>>>(f, L, B, labels, lmask, add);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int lm_gather(int* states, double* weights, float* add, const int* src_states, const double* src_weights,
              const float* src_add, const int* idx, int Rn, int V, cudaStream_t stream) {
  if (Rn <= 0) return 0;
  lm_gather_kernel<<<Rn, 128, 0, stream>>>(states, weights, add, src_states, src_weights, src_add, idx, Rn, V);
  LVSR_LAUNCH_CHECK();
  return 0;
}

}  // namespace lvsr
