// Task loss estimation (criterion mse_gain / mse_reward): the reward and gain matrices of RewardOp
// (lvsr/ops.py:236-294 over lvsr/error_rate.py:11-112) and the losses of RewardRegressionEmitter.cost
// (lvsr/bricks/__init__.py:135-184).
//
// tle_reward_kernel, one CTA per utterance, integer arithmetic throughout:
//   1. g = groundtruth cut after its first eos (none: the utterance is reported through the status word),
//      y = prediction cut the same way (none: all of it).
//   2. D[i, j] = edit distance of g[:i] and y[:j] for i <= len(g), j < len(y), an anti-diagonal wavefront over three
//      diagonals in shared memory; every cell also goes to the utterance's column-major scratch in global memory.
//   3. Per column j (one warp): opt = min_i D[i, j]; R[j, c] = -min(opt + 1, min over i < len(g), g[i] = c of D[i, j]);
//      R[j, eos] = -D[len(g) - 1, j].
//   4. G[0] = R[0], G[j] = R[j] - R[j - 1, y[j - 1]]; rows j >= len(y) hold reward -1 and gain -1000.
#include "kernels.h"
#include "lvsr_b200.h"

namespace lvsr {

namespace {

constexpr int TLE_THREADS = 256, TLE_WARPS = TLE_THREADS / 32, TLE_VMAX = 128;

struct TleArgs {
  const long long* g;      // [Lg, B]
  const long long* y;      // [L, B]
  int Lg, L, B, V, eos;
  int* dist;               // [B][L][Lg + 1]
  float* rewards;          // [L, B, V]
  float* gains;            // [L, B, V]
  unsigned* status;
};

__global__ void __launch_bounds__(TLE_THREADS) tle_reward_kernel(TleArgs a) {
  extern __shared__ int sm[];
  const int Lg = a.Lg, L = a.L, B = a.B, V = a.V, ld = Lg + 1;
  int* g = sm;                         // [Lg]
  int* y = g + Lg;                     // [L]
  int* pick = y + L;                   // [L]       R[j, y[j]]
  int* diag = pick + L;                // [3][Lg + 1]
  int* chr = diag + 3 * ld;            // [TLE_WARPS][TLE_VMAX]
  __shared__ int g_eos, y_eos;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) { g_eos = Lg; y_eos = L; }
  __syncthreads();
  for (int i = tid; i < Lg; i += TLE_THREADS) {
    const long long v = a.g[(long long)i * B + b];
    g[i] = (int)v;
    if (v == a.eos) atomicMin(&g_eos, i);
  }
  for (int j = tid; j < L; j += TLE_THREADS) {
    const long long v = a.y[(long long)j * B + b];
    y[j] = (int)v;
    if (v == a.eos) atomicMin(&y_eos, j);
  }
  __syncthreads();
  if (g_eos == Lg) {                   // reward_matrix: "Last character of the groundtruth must be EOS"
    if (tid == 0) atomicMin(a.status, (unsigned)b);
    return;
  }
  const int gl = g_eos + 1, yl = min(y_eos + 1, L);
  int* D = a.dist + (long long)b * L * ld;

  // 2. wavefront: diagonal d holds the cells i + j = d, indexed by i; D[i-1, j] and D[i, j-1] are on d - 1
  for (int d = 0; d < gl + yl; ++d) {
    int* cur = diag + (d % 3) * ld;
    const int* p1 = diag + ((d + 2) % 3) * ld;
    const int* p2 = diag + ((d + 1) % 3) * ld;
    const int i_lo = max(0, d - (yl - 1)), i_hi = min(gl, d);
    for (int i = i_lo + tid; i <= i_hi; i += TLE_THREADS) {
      const int j = d - i;
      int v;
      if (i == 0) v = j;
      else if (j == 0) v = i;
      else v = min(min(p1[i - 1], p1[i]) + 1, p2[i - 1] + (g[i - 1] != y[j - 1] ? 1 : 0));
      cur[i] = v;
      D[(long long)j * ld + i] = v;
    }
    __syncthreads();
  }

  // 3. rewards, one warp per column
  int* row = chr + warp * TLE_VMAX;
  for (int j = warp; j < yl; j += TLE_WARPS) {
    const int* col = D + (long long)j * ld;
    int opt = 0x7fffffff;
    for (int i = lane; i <= gl; i += 32) opt = min(opt, col[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) opt = min(opt, __shfl_xor_sync(0xffffffffu, opt, o));
    for (int c = lane; c < V; c += 32) row[c] = opt + 1;
    __syncwarp();
    for (int i = lane; i < gl; i += 32)
      if (g[i] >= 0 && g[i] < V) atomicMin(&row[g[i]], col[i]);
    __syncwarp();
    if (lane == 0) row[a.eos] = col[gl - 1];
    __syncwarp();
    float* out = a.rewards + ((long long)j * B + b) * V;
    for (int c = lane; c < V; c += 32) out[c] = (float)(-row[c]);
    if (lane == 0) pick[j] = (y[j] >= 0 && y[j] < V) ? -row[y[j]] : 0;
    __syncwarp();
  }
  __syncthreads();

  // 4. gains, and the rows past the prediction's eos
  for (long long e = tid; e < (long long)L * V; e += TLE_THREADS) {
    const int j = (int)(e / V), c = (int)(e % V);
    const long long o = ((long long)j * B + b) * V + c;
    if (j < yl) {
      a.gains[o] = a.rewards[o] - (j ? (float)pick[j - 1] : 0.f);
    } else {
      a.rewards[o] = -1.f;
      a.gains[o] = -1000.f;
    }
  }
}

// One warp per utterance, steps in order (the mse_reward cumulative sum runs over time).
__global__ void __launch_bounds__(256) tle_loss_kernel(int criterion, const float* neg_readouts, const float* rewards,
                                                       const float* gains, const long long* y, const float* lmask,
                                                       int L, int B, int V, float min_reward, float* costs) {
  const int lane = threadIdx.x & 31, b = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (b >= B) return;
  float cum = 0.f;                     // sum_{s <= t} of the predicted gains of the picked symbols, in float32
  for (int t = 0; t < L; ++t) {
    const long long r = (long long)t * B + b;
    const float* x = neg_readouts + r * V;
    if (criterion == LVSR_TLE_REWARD && t > 0) {
      const long long s = y[r];
      cum += (s >= 0 && s < V) ? -x[s] : 0.f;
    }
    double sum = 0.0;
    for (int v = lane; v < V; v += 32) {
      double d;
      if (criterion == LVSR_TLE_GAIN) d = (double)(-x[v]) - fmax((double)gains[r * V + v], (double)min_reward);
      else d = (double)(-x[v] + cum) - (double)rewards[r * V + v];
      sum += d * d;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) costs[r] = (float)sum * (lmask ? lmask[r] : 1.f);
  }
}

// gscale times the gradient of tle_loss_kernel's costs with respect to the readouts r = -neg_readouts, one warp per
// utterance.  mse_gain: 2 m_t (r - max(G, min_reward)).  mse_reward: with d_t = r_t + cum_t - R_t, 2 m_t d_t, and the
// picked readout r[t, y_t] (t >= 1) sits in cum_{t'} of every step t' >= t, so it also receives sum_{t' >= t} 2 m_t'
// sum_v d_t': a second, reverse-time walk over the per-step sums the first one leaves in row_sum [L, B].
__global__ void __launch_bounds__(256) tle_grad_kernel(int criterion, const float* neg_readouts, const float* rewards,
                                                       const float* gains, const long long* y, const float* lmask,
                                                       int L, int B, int V, float min_reward, float gscale,
                                                       double* row_sum, float* dlogits) {
  const int lane = threadIdx.x & 31, b = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (b >= B) return;
  float cum = 0.f;                     // as tle_loss_kernel forms it
  for (int t = 0; t < L; ++t) {
    const long long r = (long long)t * B + b;
    const float* x = neg_readouts + r * V;
    if (criterion == LVSR_TLE_REWARD && t > 0) {
      const long long s = y[r];
      cum += (s >= 0 && s < V) ? -x[s] : 0.f;
    }
    const double w = 2.0 * (lmask ? lmask[r] : 1.f);
    double sum = 0.0;
    for (int v = lane; v < V; v += 32) {
      double d;
      if (criterion == LVSR_TLE_GAIN) d = (double)(-x[v]) - fmax((double)gains[r * V + v], (double)min_reward);
      else d = (double)(-x[v] + cum) - (double)rewards[r * V + v];
      dlogits[r * V + v] = (float)(w * d * gscale);
      sum += d;
    }
    if (criterion == LVSR_TLE_REWARD) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      if (lane == 0) row_sum[r] = w * sum;
    }
  }
  if (criterion != LVSR_TLE_REWARD) return;
  __syncwarp();                        // the picked entries lane 0 adds to were written by any lane
  if (lane != 0) return;
  double acc = 0.0;
  for (int t = L - 1; t >= 1; --t) {
    const long long r = (long long)t * B + b, s = y[r];
    acc += row_sum[r];
    if (s >= 0 && s < V) dlogits[r * V + s] = (float)((double)dlogits[r * V + s] + acc * gscale);
  }
}

// One greedy step of RewardRegressionEmitter.emit (the arg-max of the readouts, the first on ties), one warp per row:
// out[b] = the pick, out_mask[b] = alive[b] (1 until the row has emitted eos), then alive[b] drops to 0 on an eos.
__global__ void __launch_bounds__(256) tle_greedy_pick_kernel(const float* neg_readouts, int B, int V, int eos,
                                                              float* alive, long long* out, float* out_mask) {
  const int lane = threadIdx.x & 31, b = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (b >= B) return;
  float bv = INFINITY;
  int bi = 0x7fffffff;
  for (int v = lane; v < V; v += 32) {
    const float x = neg_readouts[(long long)b * V + v];
    if (x < bv) { bv = x; bi = v; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov < bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  if (lane == 0) {
    if (bi == 0x7fffffff) bi = 0;      // a row of NaN
    const float a = alive[b];
    out[b] = bi;
    out_mask[b] = a;
    alive[b] = bi == eos ? 0.f : a;
  }
}

size_t tle_smem_bytes(int Lg, int L) { return (size_t)(Lg + 2 * L + 3 * (Lg + 1) + TLE_WARPS * TLE_VMAX) * sizeof(int); }

}  // namespace

size_t tle_dist_ints(int Lg, int L, int B) { return (size_t)B * L * (Lg + 1); }

int tle_matrices(const long long* groundtruth, int Lg, const long long* prediction, int L, int B, int V, int eos,
                 int* dist, float* rewards, float* gains, unsigned* status, cudaStream_t stream) {
  ProfScope prof("tle_reward", stream);
  if (B <= 0 || L <= 0) return 0;
  LVSR_CHECK(Lg > 0 && V >= 1 && V <= TLE_VMAX && eos >= 0 && eos < V, "tle: bad shapes (Lg %d, V %d, eos %d)", Lg, V, eos);
  const size_t smem = tle_smem_bytes(Lg, L);
  LVSR_CHECK(smem <= 200 * 1024, "tle: labels of %d and %d symbols do not fit the reward kernel", Lg, L);
  static size_t configured[LVSR_MAX_DEVICES] = {0};
  const int dev = current_device();
  if (smem > configured[dev] && smem > 48 * 1024) {
    LVSR_CUDA_OK(cudaFuncSetAttribute(tle_reward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured[dev] = smem;
  }
  TleArgs a = {groundtruth, prediction, Lg, L, B, V, eos, dist, rewards, gains, status};
  tle_reward_kernel<<<B, TLE_THREADS, smem, stream>>>(a);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int tle_loss(int criterion, const float* neg_readouts, const float* rewards, const float* gains,
             const long long* prediction, const float* lmask, int L, int B, int V, float min_reward, float* costs,
             cudaStream_t stream) {
  ProfScope prof("tle_loss", stream);
  if (B <= 0 || L <= 0) return 0;
  LVSR_CHECK(criterion == LVSR_TLE_GAIN || criterion == LVSR_TLE_REWARD, "tle: unknown loss %d", criterion);
  tle_loss_kernel<<<ceil_div(B, 8), 256, 0, stream>>>(criterion, neg_readouts, rewards, gains, prediction, lmask, L, B,
                                                      V, min_reward, costs);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int tle_loss_grad(int criterion, const float* neg_readouts, const float* rewards, const float* gains,
                  const long long* prediction, const float* lmask, int L, int B, int V, float min_reward, float gscale,
                  double* row_sum, float* dlogits, cudaStream_t stream) {
  ProfScope prof("tle_grad", stream);
  if (B <= 0 || L <= 0) return 0;
  LVSR_CHECK(criterion == LVSR_TLE_GAIN || criterion == LVSR_TLE_REWARD, "tle: unknown loss %d", criterion);
  tle_grad_kernel<<<ceil_div(B, 8), 256, 0, stream>>>(criterion, neg_readouts, rewards, gains, prediction, lmask, L, B,
                                                      V, min_reward, gscale, row_sum, dlogits);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int tle_greedy_pick(const float* neg_readouts, int B, int V, int eos, float* alive, long long* out, float* out_mask,
                    cudaStream_t stream) {
  if (B <= 0) return 0;
  tle_greedy_pick_kernel<<<ceil_div(B, 8), 256, 0, stream>>>(neg_readouts, B, V, eos, alive, out, out_mask);
  LVSR_LAUNCH_CHECK();
  return 0;
}

}  // namespace lvsr
