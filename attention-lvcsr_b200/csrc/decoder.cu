// Decoder-step dense pieces (skinny products with R <= a few hundred rows) and the
// readout tail.
//
// Replaces, per decoder step:
//   state_transformers.apply            s.W_state                    (lvsr/bricks/attention.py:103-104)
//   Distribute + GatedRecurrent step    ctx.W_d + fork(feedback) -> gates -> candidate -> blend
//                                        (B/bricks/attention.py:625-662, B/bricks/parallel.py:249-265,
//                                         B/bricks/recurrent.py:608-620)
//   RecurrentStack step (dec_stack 2)   each layer as above; layer 1 adds fork_1 of layer 0's new state
//                                        (B/bricks/recurrent.py:925-950)
// and, once per sequence / search step, Readout.readout + SoftmaxEmitter
//   (B/bricks/sequence_generators.py:614-619, 780-795; lvsr/bricks/recognizer.py:298-320;
//    B/bricks/simple.py:175-181, 335-371).
//
// The products are column-parallel: a CTA owns 8 output columns for a block of 64
// rows, its 8 warps split K and meet in shared memory, the GRU non-linearities are
// fused into the epilogue.  Weights are read once per launch across the grid.
#include "kernels.h"
#include "lvsr_b200.h"

namespace lvsr {

namespace {

constexpr int DR = 64;   // rows per CTA
constexpr int DN = 8;    // columns per CTA

// post_merge activation of the readout's hidden layers (LVSR_ACT_*; Maxout is accepted there with one piece only, which
// is the identity): the same expressions as readout_kernel's
__device__ __forceinline__ float readout_act(float v, int act) {
  if (act == LVSR_ACT_RELU) return fmaxf(v, 0.f);
  if (act == LVSR_ACT_TANH) return tanhf(v);
  return v;
}

// kAct: the DENSE_ACT epilogue; the other modes are the kAct = false instantiation
template <bool kAct>
__global__ void __launch_bounds__(256) dense_kernel(DenseArgs a) {
  __shared__ __align__(16) float red[8][DR * DN];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n0 = blockIdx.x * DN, r0 = blockIdx.y * DR;
  const int rg = lane >> 1, cgp = lane & 1;
  const int c0 = n0 + cgp * 4;                 // first of 4 columns of this lane
  const int rbase = r0 + rg * 4;               // first of 4 rows of this lane

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  auto run = [&](const DenseOperand& p) {
    if (p.X == nullptr || c0 >= p.ncols) return;
    // warp `warp` owns k in [k_lo, k_hi), a multiple-of-4 aligned slice
    const int kq = (p.K / 4 + 7) / 8;          // float4 groups per warp
    const int k_lo = min(p.K, warp * kq * 4), k_hi = min(p.K, k_lo + kq * 4);
    const float* xr[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) xr[i] = p.X + (long long)min(rbase + i, a.R - 1) * p.ldx;
    int k = k_lo;
    for (; k + 4 <= k_hi; k += 4) {
      float4 xv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) xv[i] = *reinterpret_cast<const float4*>(xr[i] + k);
      float4 wv[4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wv[kk] = __ldg(reinterpret_cast<const float4*>(p.W + (long long)(k + kk) * p.ncols + c0));
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float xs[4] = {xv[i].x, xv[i].y, xv[i].z, xv[i].w};
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          acc[i][0] = fmaf(xs[kk], wv[kk].x, acc[i][0]);
          acc[i][1] = fmaf(xs[kk], wv[kk].y, acc[i][1]);
          acc[i][2] = fmaf(xs[kk], wv[kk].z, acc[i][2]);
          acc[i][3] = fmaf(xs[kk], wv[kk].w, acc[i][3]);
        }
      }
    }
  };
  run(a.op[0]);
  run(a.op[1]);
  run(a.op[2]);

#pragma unroll
  for (int i = 0; i < 4; ++i)
    *reinterpret_cast<float4*>(&red[warp][(rg * 4 + i) * DN + cgp * 4]) =
        make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
  __syncthreads();

  for (int o = tid; o < DR * DN; o += 256) {
    const int rl = o / DN, cl = o % DN;
    const int r = r0 + rl, c = n0 + cl;
    if (r >= a.R || c >= a.N) continue;
    float v = 0.f;
#pragma unroll
    for (int wq = 0; wq < 8; ++wq) v += red[wq][o];
    if (a.add) {
      long long ar = a.arow ? a.arow[r] : (long long)r;
      if (a.arow && a.add_rows > 0) ar = ar < 0 ? 0 : (ar > a.add_rows - 1 ? a.add_rows - 1 : ar);
      v += a.add[ar * a.N + c];
    }
    if constexpr (kAct) {
      a.out[(long long)r * a.N + c] = readout_act(v + a.bias[c], a.act);
    } else if (a.mode == DENSE_PLAIN) {
      a.out[(long long)r * a.N + c] = v;
    } else if (a.mode == DENSE_GATES) {
      const int C = a.C;
      if (c < C) {
        a.z[(long long)r * C + c] = sigmoidf_acc(v);
      } else if (c < 2 * C) {
        const int uu = c - C;
        a.hr[(long long)r * C + uu] = a.s[(long long)r * a.ld_s + uu] * sigmoidf_acc(v);
      } else {
        a.ai[(long long)r * C + (c - 2 * C)] = v;
      }
    } else {  // DENSE_CAND
      const int C = a.C;
      const float cand = tanhf_acc(v);
      const float z = a.z[(long long)r * C + c];
      const float sold = a.s[(long long)r * a.ld_s + c];
      float sn = cand * z + sold * (1.f - z);
      if (a.rmask) {
        const float m = a.rmask[r];
        sn = m * sn + (1.f - m) * sold;
      }
      a.out[(long long)r * a.ld_out + c] = sn;
    }
  }
}

// log_softmax over the row's V entries, 4 per lane (entries >= V are -inf and stay so)
__device__ __forceinline__ void warp_log_softmax(float (&x)[4], int lane, int V) {
  float mx = -INFINITY;
#pragma unroll
  for (int q = 0; q < 4; ++q) mx = fmaxf(mx, x[q]);
  mx = warp_max(mx);
  float se = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q)
    if (lane + q * 32 < V) se += expf(x[q] - mx);
  const float lse = logf(warp_sum(se));
#pragma unroll
  for (int q = 0; q < 4; ++q) x[q] = (x[q] - mx) - lse;
}

// ShallowFusionReadout.readout + LMEmitter.costs / cost (lvsr/bricks/language_models.py), in float32 like the reference
__device__ __forceinline__ void readout_fused(const ReadoutArgs& a, int r, int lane, const float (&logit)[4]) {
  float x[4], l[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int v = lane + q * 32;
    x[q] = v < a.V ? a.am_beta * logit[q] : -INFINITY;
    l[q] = v < a.V ? -a.lm_add[(long long)r * a.V + v] : -INFINITY;
  }
  if (a.norm_am) warp_log_softmax(x, lane, a.V);
  if (a.norm_lm) warp_log_softmax(l, lane, a.V);
#pragma unroll
  for (int q = 0; q < 4; ++q) x[q] = lane + q * 32 < a.V ? x[q] + a.lm_weight * l[q] : -INFINITY;
  if (a.norm_tot) warp_log_softmax(x, lane, a.V);
  const long long lab = a.labels ? a.labels[r] : -1;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int v = lane + q * 32;
    if (v < a.V) {
      float cost = -x[q];
      if (a.poison && *a.poison != 0u) cost = __int_as_float(0x7fc00000);
      if (a.costs_all) a.costs_all[(long long)r * a.V + v] = cost;
      if (a.costs_picked && v == lab) a.costs_picked[r] = cost * (a.lmask ? a.lmask[r] : 1.f);
    }
  }
}

// One warp per row.  kTle: RewardRegressionEmitter.costs (lvsr/bricks/__init__.py:194-196), the costs are -readouts.
// kTleLm (with kTle, a.lm_add set): those readouts go through ShallowFusionReadout first, as the log-likelihood
// instantiation's fused rows do (lvsr/bricks/recognizer.py:285-297, 323-338: only the SoftmaxEmitter is swapped for
// LMEmitter, so the task-loss emitter's costs are -x of the fused x).  An instantiation of its own, so that the two
// emitters' paths without a language model keep their code.
template <bool kTle, bool kTleLm = false>
__global__ void __launch_bounds__(256) readout_kernel(ReadoutArgs a) {
  extern __shared__ float sh[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = blockIdx.x * 8 + warp;
  const int H = a.Cpm / a.pieces;
  float* hid = sh + (size_t)warp * H;
  if (r < a.R) {
    const float* mr = a.merged + (long long)r * a.Cpm;
    for (int j = lane; j < H; j += 32) {
      float v;
      if (a.act == LVSR_ACT_MAXOUT) {
        v = -INFINITY;                                           // Maxout: adjacent pieces
        for (int p = 0; p < a.pieces; ++p) v = fmaxf(v, mr[j * a.pieces + p] + a.b_pm[j * a.pieces + p]);
      } else {
        v = mr[j] + a.b_pm[j];
        if (a.act == LVSR_ACT_RELU) v = fmaxf(v, 0.f);
        else if (a.act == LVSR_ACT_TANH) v = tanhf(v);
      }
      hid[j] = v;
    }
  }
  __syncwarp();
  if (r >= a.R) return;
  // logits for v = lane, lane + 32, ... (V <= 128)
  float logit[4];
  float vmax = -INFINITY;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int v = lane + q * 32;
    float s = -INFINITY;
    if (v < a.V) {
      s = a.bo[v];
      for (int j = 0; j < H; ++j) s = fmaf(hid[j], __ldg(a.Wo + (long long)j * a.V + v), s);
    }
    logit[q] = s;
    vmax = fmaxf(vmax, s);
  }
  if constexpr (kTleLm) {
    readout_fused(a, r, lane, logit);
    return;
  }
  if constexpr (kTle) {
    const long long lab = a.labels ? a.labels[r] : -1;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int v = lane + q * 32;
      if (v < a.V) {
        float cost = -logit[q];
        if (a.poison && *a.poison != 0u) cost = __int_as_float(0x7fc00000);
        if (a.costs_all) a.costs_all[(long long)r * a.V + v] = cost;
        if (a.costs_picked && v == lab) a.costs_picked[r] = cost * (a.lmask ? a.lmask[r] : 1.f);
      }
    }
    return;
  }
  vmax = warp_max(vmax);
  if (a.lm_add) {
    readout_fused(a, r, lane, logit);
    return;
  }
  float se = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q)
    if (lane + q * 32 < a.V) se += expf(logit[q] - vmax);
  se = warp_sum(se);
  const float lse = logf(se);
  const long long lab = a.labels ? a.labels[r] : -1;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int v = lane + q * 32;
    if (v < a.V) {
      float cost = -((logit[q] - vmax) - lse);
      if (a.poison && *a.poison != 0u) cost = __int_as_float(0x7fc00000);   // producer kernel reported a failed launch
      if (a.costs_all) a.costs_all[(long long)r * a.V + v] = cost;
      if (a.costs_picked && v == lab) a.costs_picked[r] = cost * (a.lmask ? a.lmask[r] : 1.f);
    }
  }
}

__global__ void fill_f32_kernel(float* p, long long n, float v) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void fill_i64_kernel(long long* p, long long n, long long v) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void broadcast_rows_kernel(float* dst, const float* src, long long total, int N) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i % N];
}
__global__ void add_bias_rows_kernel(float* dst, const float* src, const float* bias, long long total, int N) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i] + bias[i % N];
}
__global__ void onehot_rows_kernel(float* dst, long long total, int N) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) dst[i] = (i % N == 0) ? 1.f : 0.f;
}
__global__ void add_i64_kernel(long long* dst, const long long* src, int n, long long inc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[i] + inc;
}
__global__ void gather_time_kernel(float* dst, const float* src, int Tout, int k, long long row_elems) {
  const long long total = (long long)Tout * row_elems;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / row_elems, e = i % row_elems;
    dst[i] = src[t * k * row_elems + e];
  }
}

__global__ void gather_rows_kernel(float* dst, const float* src, const int* idx, long long total, int N) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    dst[i] = src[(long long)idx[i / N] * N + i % N];
}
__global__ void gather_i64_kernel(long long* dst, const long long* src, const int* idx, int n, long long inc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[idx[i]] + inc;
}

// BeamSearch._smallest (B/search.py:220-242) for every utterance of a batched search: the k smallest entries of
// cost_so_far[r] + neglogp[r, v] over the segment's rows, in increasing order (ties: smaller flat index first).
// One CTA per segment; the candidate table (width x V <= k x 128 floats) lives in shared memory and k rounds of a
// block-wide arg-min pick the winners.  top_count = -1 flags a non-finite log-probability (the reference asserts).
__global__ void __launch_bounds__(256) segment_topk_kernel(const float* neglogp, const float* cost_so_far, const int* seg_start,
                                                           int V, int k, int* top_parent, int* top_symbol, float* top_cost,
                                                           int* top_count) {
  extern __shared__ float cand[];
  __shared__ float rv[8];
  __shared__ int ri[8];
  __shared__ int bad;
  const int sg = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int r0 = seg_start[sg], width = seg_start[sg + 1] - r0, n = width * V;
  if (tid == 0) bad = 0;
  __syncthreads();
  for (int i = tid; i < n; i += 256) {
    const float lp = neglogp[(long long)r0 * V + i];
    if (!isfinite(lp)) bad = 1;
    cand[i] = cost_so_far[r0 + i / V] + lp;
  }
  __syncthreads();
  const int take = min(k, n);
  for (int round = 0; round < take; ++round) {
    float bv = INFINITY;
    int bi = 0x7fffffff;
    for (int i = tid; i < n; i += 256) {
      const float v = cand[i];
      if (v < bv) { bv = v; bi = i; }           // strided scan keeps the smallest index among equal values per thread
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov < bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { rv[warp] = bv; ri[warp] = bi; }
    __syncthreads();
    if (tid == 0) {
      for (int q = 1; q < 8; ++q)
        if (rv[q] < rv[0] || (rv[q] == rv[0] && ri[q] < ri[0])) { rv[0] = rv[q]; ri[0] = ri[q]; }
      const int idx = ri[0];
      if (idx != 0x7fffffff) {
        top_parent[sg * k + round] = r0 + idx / V;
        top_symbol[sg * k + round] = idx % V;
        top_cost[sg * k + round] = rv[0];
        cand[idx] = INFINITY;
      } else {                                  // every remaining candidate is +inf / NaN
        top_parent[sg * k + round] = -1;
      }
    }
    __syncthreads();
  }
  if (tid == 0) top_count[sg] = bad ? -1 : take;
}

inline int grid_for(long long n) { return (int)std::min<long long>(2048, std::max<long long>(1, (n + 255) / 256)); }

}  // namespace

int dense_step(const DenseArgs& a, cudaStream_t stream) {
  ProfScope prof("dense", stream);
  if (a.R <= 0) return 0;
  LVSR_CHECK(a.N % 4 == 0, "dense_step: N=%d is not a multiple of 4", a.N);
  for (const DenseOperand& p : a.op)
    LVSR_CHECK(!p.X || (p.K % 4 == 0 && p.ldx % 4 == 0 && p.ncols % 4 == 0),
               "dense_step: dimensions and strides must be multiples of 4 (K=%d ldx=%d ncols=%d)", p.K, p.ldx, p.ncols);
  LVSR_CHECK(a.mode != DENSE_ACT || a.bias, "dense_step: DENSE_ACT without a bias");
  dim3 grid(ceil_div(a.N, DN), ceil_div(a.R, DR));
  if (a.mode == DENSE_ACT) dense_kernel<true><<<grid, 256, 0, stream>>>(a);
  else dense_kernel<false><<<grid, 256, 0, stream>>>(a);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int readout_costs(const ReadoutArgs& a, cudaStream_t stream) {
  ProfScope prof("readout", stream);
  if (a.R <= 0) return 0;
  LVSR_CHECK(a.V <= 128, "readout: num_phonemes %d > 128 unsupported", a.V);
  LVSR_CHECK(a.pieces >= 1 && a.Cpm % a.pieces == 0, "readout: bad maxout pieces");
  const size_t smem = readout_smem_bytes(a.Cpm / a.pieces);
  LVSR_CHECK(smem <= READOUT_SMEM_LIMIT, "readout: post_merge_dim too large");
  if (a.tle && a.lm_add) readout_kernel<true, true><<<ceil_div(a.R, 8), 256, smem, stream>>>(a);
  else if (a.tle) readout_kernel<true><<<ceil_div(a.R, 8), 256, smem, stream>>>(a);
  else readout_kernel<false><<<ceil_div(a.R, 8), 256, smem, stream>>>(a);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int fill_f32(float* p, long long n, float v, cudaStream_t stream) {
  if (n <= 0) return 0;
  fill_f32_kernel<<<grid_for(n), 256, 0, stream>>>(p, n, v);
  LVSR_LAUNCH_CHECK();
  return 0;
}
int fill_i64(long long* p, long long n, long long v, cudaStream_t stream) {
  if (n <= 0) return 0;
  fill_i64_kernel<<<grid_for(n), 256, 0, stream>>>(p, n, v);
  LVSR_LAUNCH_CHECK();
  return 0;
}
int broadcast_rows(float* dst, const float* src, int R, int N, cudaStream_t stream) {
  const long long total = (long long)R * N;
  if (total <= 0) return 0;
  broadcast_rows_kernel<<<grid_for(total), 256, 0, stream>>>(dst, src, total, N);
  LVSR_LAUNCH_CHECK();
  return 0;
}
int add_bias_rows(float* dst, const float* src, const float* bias, int R, int N, cudaStream_t stream) {
  const long long total = (long long)R * N;
  if (total <= 0) return 0;
  add_bias_rows_kernel<<<grid_for(total), 256, 0, stream>>>(dst, src, bias, total, N);
  LVSR_LAUNCH_CHECK();
  return 0;
}
int onehot_rows(float* dst, int R, int N, cudaStream_t stream) {
  const long long total = (long long)R * N;
  if (total <= 0) return 0;
  onehot_rows_kernel<<<grid_for(total), 256, 0, stream>>>(dst, total, N);
  LVSR_LAUNCH_CHECK();
  return 0;
}
int gather_rows(float* dst, const float* src, const int* idx, int Rn, int N, cudaStream_t stream) {
  const long long total = (long long)Rn * N;
  if (total <= 0) return 0;
  gather_rows_kernel<<<grid_for(total), 256, 0, stream>>>(dst, src, idx, total, N);
  LVSR_LAUNCH_CHECK();
  return 0;
}
int gather_i64(long long* dst, const long long* src, const int* idx, int Rn, long long inc, cudaStream_t stream) {
  if (Rn <= 0) return 0;
  gather_i64_kernel<<<ceil_div(Rn, 256), 256, 0, stream>>>(dst, src, idx, Rn, inc);
  LVSR_LAUNCH_CHECK();
  return 0;
}
int segment_topk(const float* neglogp, const float* cost_so_far, const int* seg_start, int nseg, int V, int k,
                 int* top_parent, int* top_symbol, float* top_cost, int* top_count, cudaStream_t stream) {
  if (nseg <= 0) return 0;
  const size_t smem = (size_t)k * V * sizeof(float);        // a segment never holds more than k rows
  LVSR_CHECK(smem <= 200 * 1024, "beam search: beam_size %d x %d symbols does not fit the selection kernel", k, V);
  static size_t configured[LVSR_MAX_DEVICES] = {0};
  const int dev = current_device();
  if (smem > configured[dev] && smem > 48 * 1024) {
    LVSR_CUDA_OK(cudaFuncSetAttribute(segment_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured[dev] = smem;
  }
  segment_topk_kernel<<<nseg, 256, smem, stream>>>(neglogp, cost_so_far, seg_start, V, k, top_parent, top_symbol, top_cost, top_count);
  LVSR_LAUNCH_CHECK();
  return 0;
}
int add_i64(long long* dst, const long long* src, int n, long long inc, cudaStream_t stream) {
  if (n <= 0) return 0;
  add_i64_kernel<<<ceil_div(n, 256), 256, 0, stream>>>(dst, src, n, inc);
  LVSR_LAUNCH_CHECK();
  return 0;
}
int gather_time_subsample(float* dst, const float* src, int Tout, int k, long long row_elems, cudaStream_t stream) {
  const long long total = (long long)Tout * row_elems;
  if (total <= 0) return 0;
  gather_time_kernel<<<grid_for(total), 256, 0, stream>>>(dst, src, Tout, k, row_elems);
  LVSR_LAUNCH_CHECK();
  return 0;
}

}  // namespace lvsr
