// Kernels of the training step (SURVEY.md section 8 rows a21 / f1): everything the backward pass needs
// besides the two reverse-time scans that have files of their own (bigru_bwd.cu; the decoder's
// step loop is orchestrated in train.cu out of the kernels below).
//
// Reference: theano.tensor.grad of sum(cost_matrix)/B through the graph of SURVEY.md section 9
// (lvsr/main.py:340-345; B/algorithms/__init__.py:218-225), then the step rules of
// lvsr/main.py:480-519 / B/algorithms/__init__.py:378-893.  Checked against
// oracle/lvsr_oracle_grad.py (float64 autograd + numpy step rules).
#pragma once
#include "kernels.h"
#include "lvsr_b200.h"

namespace lvsr {
namespace train {

// ------------------------------------------------------------------------------------------
// C[Mo, N] (+)= A^T B over R rows:  A [R, lda] (columns m0 .. m0+Mo), B [R, ldb].
// Weight gradients (dW = X^T dY).  Split over R: grid.z CTAs each reduce a slice of rows into a
// partial tile; tn_reduce adds the partials in a fixed order (deterministic, no atomics).
// ------------------------------------------------------------------------------------------
constexpr int TN_BM = 64, TN_BN = 64, TN_BK = 16;

struct TnArgs {
  const float* A; int lda;
  const float* B; int ldb;
  int R, Mo, N;
  float* part;            // [splits][Mo][N]
  int rows_per_split;
  int vec_a, vec_b;       // rows of A / B start on 16-byte boundaries (aligned base, leading dimension % 4 == 0)
};

__global__ void __launch_bounds__(256) gemm_tn_kernel(TnArgs g) {
  __shared__ __align__(16) float As[2][TN_BK][TN_BM];
  __shared__ __align__(16) float Bs[2][TN_BK][TN_BN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int n0 = blockIdx.x * TN_BN, m0 = blockIdx.y * TN_BM;
  const int r_lo = blockIdx.z * g.rows_per_split, r_hi = min(g.R, r_lo + g.rows_per_split);
  // loaders: four consecutive columns of one row per thread for each operand (16 rows x 64 columns per tile), one
  // float4 where the row is 16-byte aligned, scalar loads otherwise (e.g. ldb = V = 63, lda = 123 features)
  const int lr = tid >> 4, lc = (tid & 15) * 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  float4 ra, rb;
  auto load = [&](int r0) {
    const int r = r0 + lr;
    ra = make_float4(0.f, 0.f, 0.f, 0.f);
    rb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < r_hi) {
      const float* ap = g.A + (long long)r * g.lda + m0 + lc;
      const float* bp = g.B + (long long)r * g.ldb + n0 + lc;
      if (g.vec_a && m0 + lc + 3 < g.Mo) ra = *reinterpret_cast<const float4*>(ap);
      else {
        if (m0 + lc + 0 < g.Mo) ra.x = ap[0];
        if (m0 + lc + 1 < g.Mo) ra.y = ap[1];
        if (m0 + lc + 2 < g.Mo) ra.z = ap[2];
        if (m0 + lc + 3 < g.Mo) ra.w = ap[3];
      }
      if (g.vec_b && n0 + lc + 3 < g.N) rb = *reinterpret_cast<const float4*>(bp);
      else {
        if (n0 + lc + 0 < g.N) rb.x = bp[0];
        if (n0 + lc + 1 < g.N) rb.y = bp[1];
        if (n0 + lc + 2 < g.N) rb.z = bp[2];
        if (n0 + lc + 3 < g.N) rb.w = bp[3];
      }
    }
  };
  auto store = [&](int buf) {
    *reinterpret_cast<float4*>(&As[buf][lr][lc]) = ra;
    *reinterpret_cast<float4*>(&Bs[buf][lr][lc]) = rb;
  };
  const int nk = (r_hi - r_lo + TN_BK - 1) / TN_BK;
  if (nk > 0) { load(r_lo); store(0); }
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load(r_lo + (kt + 1) * TN_BK);
#pragma unroll
    for (int k = 0; k < TN_BK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (kt + 1 < nk) store(buf ^ 1);
    __syncthreads();
  }
  float* out = g.part + (long long)blockIdx.z * g.Mo * g.N;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= g.Mo) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n < g.N) out[(long long)m * g.N + n] = acc[i][j];
    }
  }
}

// C[m, n] (ldc) = (accumulate ? C : 0) + scale * sum_z part[z][m][n]
__global__ void tn_reduce_kernel(const float* part, int splits, int Mo, int N, float* C, int ldc, int accumulate) {
  const long long total = (long long)Mo * N;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    float v = 0.f;
    for (int z = 0; z < splits; ++z) v += part[(long long)z * total + i];
    const int m = (int)(i / N), n = (int)(i % N);
    float* c = C + (long long)m * ldc + n;
    *c = accumulate ? (*c + v) : v;
  }
}

// out[n] (+)= sum_r X[r, n]   (bias gradients; X has leading dimension ldx)
__global__ void __launch_bounds__(256) colsum_kernel(const float* X, int R, int N, int ldx, float* out, int accumulate) {
  __shared__ float red[8][32];
  const int n = blockIdx.x * 32 + (threadIdx.x & 31), w = threadIdx.x >> 5;
  float s = 0.f;
  if (n < N)
    for (int r = w; r < R; r += 8) s += X[(long long)r * ldx + n];
  red[w][threadIdx.x & 31] = s;
  __syncthreads();
  if (w == 0 && n < N) {
    float v = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) v += red[q][threadIdx.x];
    out[n] = accumulate ? out[n] + v : v;
  }
}

// dst[n, k] = src[k, n]
__global__ void transpose_kernel(const float* __restrict__ src, float* __restrict__ dst, int K, int N) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = k0 + i, n = n0 + threadIdx.x;
    tile[i][threadIdx.x] = (k < K && n < N) ? src[(long long)k * N + n] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int n = n0 + i, k = k0 + threadIdx.x;
    if (n < N && k < K) dst[(long long)n * K + k] = tile[threadIdx.x][i];
  }
}

// ------------------------------------------------------------------------------------------
// Skinny product of the decoder's backward step: out[R, N] (ldo) = sum_p X_p[R, K_p] (ldx_p) . W_p[K_p, N]
// + add0 + add1, R = batch rows.  Same shape as dense_kernel (decoder.cu) with leading dimensions.
// ------------------------------------------------------------------------------------------
struct SkinnyArgs {
  const float* X[2]; int K[2]; int ldx[2]; const float* W[2];     // W_p [K_p, N] row-major (ld N)
  const float* add[2]; int lda[2];
  float* out; int ldo;
  int R, N;
  // optional column split: columns >= split go to out1 (ldo1) and take add[1] INSTEAD of add[0] (two products that share
  // the left-hand side fused into one launch); split = 0: one output, both addends
  int split; float* out1; int ldo1;
};
constexpr int SK_R = 64, SK_N = 8, SK_WARPS = 16;

// 64 rows x 8 columns per CTA, K split over 16 warps; two 4-wide k groups are in flight per iteration (the loop is
// bound by the L2 latency of its operand loads, not by the FMAs).
__global__ void __launch_bounds__(SK_WARPS * 32) skinny_kernel(SkinnyArgs a) {
  __shared__ __align__(16) float red[SK_WARPS][SK_R * SK_N];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n0 = blockIdx.x * SK_N, r0 = blockIdx.y * SK_R;
  const int rg = lane >> 1, cgp = lane & 1;
  const int c0 = n0 + cgp * 4, rbase = r0 + rg * 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll
  for (int p = 0; p < 2; ++p) {
    if (a.X[p] == nullptr || c0 >= a.N) continue;
    const int K = a.K[p];
    const int kq = (K / 4 + SK_WARPS - 1) / SK_WARPS;
    const int k_lo = min(K, warp * kq * 4), k_hi = min(K, k_lo + kq * 4);
    const float* xr[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) xr[i] = a.X[p] + (long long)min(rbase + i, a.R - 1) * a.ldx[p];
    const float* wp = a.W[p] + c0;
    auto fma16 = [&](const float4 (&xv)[4], const float4 (&wv)[4]) {
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
    };
    int k = k_lo;
    for (; k + 8 <= k_hi; k += 8) {
      float4 xa[4], wa[4], xb[4], wb[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { xa[i] = *reinterpret_cast<const float4*>(xr[i] + k); xb[i] = *reinterpret_cast<const float4*>(xr[i] + k + 4); }
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        wa[kk] = __ldg(reinterpret_cast<const float4*>(wp + (long long)(k + kk) * a.N));
        wb[kk] = __ldg(reinterpret_cast<const float4*>(wp + (long long)(k + 4 + kk) * a.N));
      }
      fma16(xa, wa);
      fma16(xb, wb);
    }
    for (; k + 4 <= k_hi; k += 4) {
      float4 xa[4], wa[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) xa[i] = *reinterpret_cast<const float4*>(xr[i] + k);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wa[kk] = __ldg(reinterpret_cast<const float4*>(wp + (long long)(k + kk) * a.N));
      fma16(xa, wa);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
    *reinterpret_cast<float4*>(&red[warp][(rg * 4 + i) * SK_N + cgp * 4]) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
  __syncthreads();
  for (int o = tid; o < SK_R * SK_N; o += SK_WARPS * 32) {
    const int rl = o / SK_N, cl = o % SK_N;
    const int r = r0 + rl, c = n0 + cl;
    if (r >= a.R || c >= a.N) continue;
    float v = 0.f;
#pragma unroll
    for (int wq = 0; wq < SK_WARPS; ++wq) v += red[wq][o];
    if (a.split > 0) {
      if (c < a.split) {
        if (a.add[0]) v += a.add[0][(long long)r * a.lda[0] + c];
        a.out[(long long)r * a.ldo + c] = v;
      } else {
        if (a.add[1]) v += a.add[1][(long long)r * a.lda[1] + c - a.split];
        a.out1[(long long)r * a.ldo1 + c - a.split] = v;
      }
    } else {
      if (a.add[0]) v += a.add[0][(long long)r * a.lda[0] + c];
      if (a.add[1]) v += a.add[1][(long long)r * a.lda[1] + c];
      a.out[(long long)r * a.ldo + c] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------
// Readout + emitter backward, one warp per (step, row): recomputes the forward of readout_kernel (decoder.cu) and
// emits hid (post-activation) and dmerged (through Linear^T and Maxout / ReLU / Tanh / Identity and the Bias) from
// dlogits.  SoftmaxEmitter (kTle false) forms dlogits = (softmax - onehot(label)) * mask * gscale itself;
// RewardRegressionEmitter (kTle true) reads the dlogits tle_loss_grad wrote.
// ------------------------------------------------------------------------------------------
struct ReadoutBwdArgs {
  const float* merged;     // [R, Cpm]  states.W_ms + ctx.W_mc
  const float* b_pm; const float* Wo; const float* bo;
  int R, Cpm, pieces, V, act;
  const long long* labels; const float* lmask;
  float gscale;
  float* hid;              // [R, Cpm/pieces]
  float* dlogits;          // [R, V]: written (kTle false) or read (kTle true)
  float* dmerged;          // [R, Cpm]
};

template <bool kTle>
__global__ void __launch_bounds__(256) readout_bwd_kernel(ReadoutBwdArgs a) {
  extern __shared__ float sh[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = blockIdx.x * 8 + warp;
  const int H = a.Cpm / a.pieces;
  float* hid = sh + (size_t)warp * (H + 128);
  float* dl = hid + H;                 // [V <= 128]
  if (r >= a.R) return;
  const float* mr = a.merged + (long long)r * a.Cpm;
  for (int j = lane; j < H; j += 32) {
    float v;
    if (a.act == LVSR_ACT_MAXOUT) {
      v = -INFINITY;
      for (int p = 0; p < a.pieces; ++p) v = fmaxf(v, mr[j * a.pieces + p] + a.b_pm[j * a.pieces + p]);
    } else {
      v = mr[j] + a.b_pm[j];
      if (a.act == LVSR_ACT_RELU) v = fmaxf(v, 0.f);
      else if (a.act == LVSR_ACT_TANH) v = tanhf(v);
    }
    hid[j] = v;
    a.hid[(long long)r * H + j] = v;
  }
  __syncwarp();
  if constexpr (kTle) {
    for (int v = lane; v < a.V; v += 32) dl[v] = a.dlogits[(long long)r * a.V + v];
  } else {
    float logit[4], vmax = -INFINITY;
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
    vmax = warp_max(vmax);
    float se = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (lane + q * 32 < a.V) se += expf(logit[q] - vmax);
    se = warp_sum(se);
    const long long lab = a.labels[r];
    const float w = (a.lmask ? a.lmask[r] : 1.f) * a.gscale;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int v = lane + q * 32;
      if (v < a.V) {
        const float g = (expf(logit[q] - vmax) / se - (v == lab ? 1.f : 0.f)) * w;
        dl[v] = g;
        a.dlogits[(long long)r * a.V + v] = g;
      }
    }
  }
  __syncwarp();
  // dhid[j] = sum_v dlogits[v] Wo[j, v]; route through the activation
  for (int j = lane; j < H; j += 32) {
    float dh = 0.f;
    for (int v = 0; v < a.V; ++v) dh = fmaf(dl[v], __ldg(a.Wo + (long long)j * a.V + v), dh);
    if (a.act == LVSR_ACT_MAXOUT) {
      int best = 0;
      float bv = -INFINITY;
      for (int p = 0; p < a.pieces; ++p) {          // first maximum wins (theano max gradient: eq to max; ties are measure-zero)
        const float x = mr[j * a.pieces + p] + a.b_pm[j * a.pieces + p];
        if (x > bv) { bv = x; best = p; }
      }
      for (int p = 0; p < a.pieces; ++p) a.dmerged[(long long)r * a.Cpm + j * a.pieces + p] = (p == best) ? dh : 0.f;
    } else {
      float g = dh;
      if (a.act == LVSR_ACT_RELU) g = (mr[j] + a.b_pm[j] > 0.f) ? dh : 0.f;
      else if (a.act == LVSR_ACT_TANH) g = dh * (1.f - hid[j] * hid[j]);
      a.dmerged[(long long)r * a.Cpm + j] = g;
    }
  }
}

// ------------------------------------------------------------------------------------------
// Bulk recomputation of the decoder GRU's gate values for all L steps at once (the forward scan
// keeps only states and glimpses): G [R, 3C] holds ctx.Wd + s.Wg (gate columns) on entry.
//   gates: adds fork(feedback(label)), Z = sigma(G[:, :C]), Rg = sigma(G[:, C:2C]), HR = S_prev * Rg,
//          A = G[:, 2C:] + FF[:, 2C:] stays in G's third block
//   cand:  Cc = tanh(Cpre + A)
// ------------------------------------------------------------------------------------------
__global__ void dec_gates_kernel(float* G, const float* FF, const long long* labels, const float* S_prev, int R, int C,
                                 float* Z, float* Rg, float* HR) {
  const long long total = (long long)R * 3 * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / (3 * C)), c = (int)(i % (3 * C));
    const float v = G[i] + FF[labels[r] * 3 * C + c];
    if (c < C) Z[(long long)r * C + c] = 1.f / (1.f + expf(-v));
    else if (c < 2 * C) {
      const float g = 1.f / (1.f + expf(-v));
      Rg[(long long)r * C + c - C] = g;
      HR[(long long)r * C + c - C] = S_prev[(long long)r * C + c - C] * g;
    } else G[i] = v;
  }
}
__global__ void dec_cand_kernel(const float* Cpre, const float* G, int R, int C, float* Cc) {
  const long long total = (long long)R * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / C), c = (int)(i % C);
    Cc[i] = tanhf(Cpre[i] + G[(long long)r * 3 * C + 2 * C + c]);
  }
}

// decoder GRU step backward, element-wise parts (B/bricks/recurrent.py:608-620 differentiated; see bigru_bwd.cu)
//  a: ds (grad of s_i) -> dG[:, 2C:] = dA, dG[:, :C] = dGz, keep = (1-m) ds + m ds (1-z)
__global__ void dec_bwd_a_kernel(const float* ds, const float* Z, const float* Cc, const float* S_prev, const float* lmask,
                                 int R, int C, float* dG, float* keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * C) return;
  const int r = i / C, c = i % C;
  const float m = lmask ? lmask[r] : 1.f;
  const float z = Z[i], cc = Cc[i], h = S_prev[i], tot = ds[i];
  const float dht = m * tot;
  keep[i] = (1.f - m) * tot + dht * (1.f - z);
  dG[(long long)r * 3 * C + 2 * C + c] = dht * z * (1.f - cc * cc);
  dG[(long long)r * 3 * C + c] = dht * (cc - h) * z * (1.f - z);
}
//  b: dHR -> dG[:, C:2C] = dGr, keep += dHR * r
__global__ void dec_bwd_b_kernel(const float* dHR, const float* Rg, const float* S_prev, int R, int C, float* dG, float* keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * C) return;
  const int r = i / C, c = i % C;
  const float g = Rg[i], d = dHR[i];
  keep[i] += d * g;
  dG[(long long)r * 3 * C + C + c] = d * S_prev[i] * g * (1.f - g);
}

// dFF[label[r], :] += dG[r, :]  -- one CTA per table row (deterministic: rows added in order)
__global__ void __launch_bounds__(256) scatter_rows_kernel(const float* dG, const long long* labels, int R, int N, float* dFF) {
  const int y = blockIdx.x;
  for (int c = threadIdx.x; c < N; c += blockDim.x) {
    float s = 0.f;
    for (int r = 0; r < R; ++r)
      if (labels[r] == y) s += dG[(long long)r * N + c];
    dFF[(long long)y * N + c] = s;
  }
}

// dH[t, b, :] += sum_i alpha_i[b, t] dctx_i[b, :]    (weighted averages, B/bricks/attention.py:256)
__global__ void __launch_bounds__(256) dh_from_ctx_kernel(const float* W_all, const float* dctx_all, int L, int B, int Tp, int E,
                                                          float* dH, int accumulate) {
  // CTA: one batch row, 8 positions; thread: one column group of E (E <= 1024: up to 4 columns per thread)
  const int b = blockIdx.y, t0 = blockIdx.x * 8;
  float acc[8][4];
#pragma unroll
  for (int q = 0; q < 8; ++q)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[q][j] = 0.f;
  __shared__ float sw[8];
  for (int i = 0; i < L; ++i) {
    if (threadIdx.x < 8) sw[threadIdx.x] = (t0 + threadIdx.x < Tp) ? W_all[((long long)i * B + b) * Tp + t0 + threadIdx.x] : 0.f;
    __syncthreads();
    const float* dc = dctx_all + ((long long)i * B + b) * E;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int e = threadIdx.x + j * 256;
      if (e < E) {
        const float d = dc[e];
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q][j] = fmaf(sw[q], d, acc[q][j]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    if (t0 + q >= Tp) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int e = threadIdx.x + j * 256;
      if (e < E) {
        float* p = dH + ((long long)(t0 + q) * B + b) * E + e;
        *p = accumulate ? *p + acc[q][j] : acc[q][j];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Attention step backward for one decoder step: 2 CTAs per batch row (halves of the window).
// Forward math: lvsr/bricks/attention.py:98-114,165-183,191-213.
// With g[t] = dctx . H[t] + carry[t] the gradient reaching alpha_i[t] and S = sum_t alpha_i[t] g[t], the energy
// gradient of each normaliser (e includes the energy bias; the window mask m is folded into alpha):
//   softmax   alpha = exp(e) m / N:        de = alpha (g - S)
//   logistic  alpha = sigma(e) m / N:      de = alpha (1 - sigma(e)) (g - S)
//   relu      alpha = max(e/1000, 0) m / N: de = m [e > 0] (g - S) / (1000 N) = (g - S) alpha / e where e > 0, else 0
// N is the same for every position of a row, so the relu rule reads 1 / (1000 N) off the alignment instead of
// re-forming the window's mask and sum.  The energy bias b enters every energy: db = sum of de.
// ------------------------------------------------------------------------------------------
constexpr int AB_NT = 512;
constexpr int AB_CS = 2;
constexpr int AB_TILE = 16;

struct AttBwdArgs {
  const float* P; const float* H; const float* maskH;      // [Tp,B,M], [Tp,B,E], [Tp,B]
  const float* q;            // [B, M]   s_{i-1} . W_s
  const float* w_prev;       // [B, Tp]  alpha_{i-1}
  const float* w_cur;        // [B, Tp]  alpha_i
  const float* ctx;          // [B, E]   weighted averages of step i
  const float* dctx;         // [B, E]
  const float* dA_in;        // [2][B][Tp] gradient of alpha_i from step i+1 (two partial buffers) or nullptr (zero)
  const int* win;            // [2]
  const float* filt; const float* Wh; const float* v;        // [K,w], [K,M], [M]
  float* dP;                 // [Tp,B,M]  accumulated in place
  float* dq_part;            // [2][B][M]
  float* dA_out;             // [2][B][Tp] gradient of alpha_{i-1}
  float* acc_v;              // [2B][M]     per-CTA partial sums over the steps
  float* acc_Wh;             // [2B][K][M]
  float* acc_filt;           // [2B][K][w]
  int B, Tp, M, E, K, n;
  const float* e_cur;        // [B, Tp]  energies of step i, bias included (logistic / relu only)
  float* acc_b;              // [2B]     per-CTA partial sums of de (logistic / relu only)
  const float* pen;          // [B, Tp]  gradient of the alignment penalty w.r.t. alpha_i, or nullptr (none)
};

// Alignment monotonicity penalty (lvsr/expressions.py:14-19) of the taped alignments W [L, B, Tp], c_i = cumsum_t w_i:
//   P = sum_b sum_{i>=1} m[i,b] sum_t max(c_i[t] - c_{i-1}[t], 0)
//   dP/dw_i[t'] = sum_{t>=t'} (m_i [c_i[t] >= c_{i-1}[t]] - m_{i+1} [c_{i+1}[t] >= c_i[t]])   (first term absent for
//   i = 0, second for i = L-1; a tie counts as 1, the gradient of Theano's maximum)
// One thread per (i, b) row: grad [L, B, Tp] = scale * dP/dw, row_sum [L * B] = the row's term of P (0 for i = 0).
__global__ void __launch_bounds__(256) penalty_grad_kernel(const float* __restrict__ W, const float* __restrict__ lmask,
                                                           int L, int B, int Tp, float scale, float* __restrict__ grad,
                                                           float* __restrict__ row_sum) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= L * B) return;
  const int i = r / B, b = r % B;
  const float* wc = W + (size_t)r * Tp;
  const float* wp = i > 0 ? wc - (size_t)B * Tp : nullptr;
  const float* wn = i + 1 < L ? wc + (size_t)B * Tp : nullptr;
  const float mi = i > 0 ? (lmask ? lmask[r] : 1.f) : 0.f;
  const float mn = wn ? (lmask ? lmask[r + B] : 1.f) : 0.f;
  float* g = grad + (size_t)r * Tp;
  float cp = 0.f, cc = 0.f, cn = 0.f, sum = 0.f;
  for (int t = 0; t < Tp; ++t) {
    cc += wc[t];
    float v = 0.f;
    if (wp) {
      cp += wp[t];
      if (cc >= cp) { v += mi; sum += cc - cp; }
    }
    if (wn) {
      cn += wn[t];
      if (cn >= cc) v -= mn;
    }
    g[t] = v;
  }
  float acc = 0.f;
  for (int t = Tp - 1; t >= 0; --t) {
    acc += g[t];
    g[t] = scale * acc;
  }
  row_sum[r] = mi * sum;
}

__host__ __device__ inline int att_bwd_kp(int K) { return K <= 12 ? 12 : 16; }     // padded row of K filter values (float4 loads)

__host__ __device__ inline size_t att_bwd_smem_floats(int M, int E, int K, int n, int tc_cap) {
  const int KP = att_bwd_kp(K);
  size_t f = 0;
  f += tc_cap + 2 * n + 8;                 // salpha
  f += 4;                                  // alignment slack
  f += (size_t)(2 * n + 1) * KP;           // sfilt [j][KP]
  f += (size_t)K * M;                      // sWh
  f += (size_t)tc_cap * KP;                // sF
  f += (size_t)tc_cap * KP;                // sdF
  f += tc_cap + 4;                         // sde
  f += (size_t)AB_TILE * M;                // sdm
  f += E;                                  // sdctx
  f += 64;                                 // block reductions
  return f + 16;
}

__device__ __forceinline__ float block_sum_512(float v, float* scratch) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < AB_NT / 32; ++i) s += scratch[i];
  return s;
}

// KP: padded filter-row length (12 or 16).  Everything indexed by the filter k is held as KP-wide float4 rows so the
// inner loops are vector shared-memory loads + FMAs; the handler column of a thread lives in registers.
// NORM: the energy normaliser (LVSR_NORM_*); it changes the energy gradient and adds the bias partial only.
template <int KP, int NORM>
__global__ void __launch_bounds__(AB_NT, 1) att_bwd_kernel(AttBwdArgs a, int tc_cap) {
  extern __shared__ __align__(16) float smem[];
  constexpr int KV = KP / 4;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.x / AB_CS, rank = blockIdx.x % AB_CS;
  const int M = a.M, E = a.E, K = a.K, n = a.n, w = 2 * n + 1, Tp = a.Tp, B = a.B;
  float* salpha = smem;
  float* sfilt = salpha + ((tc_cap + 2 * n + 8 + 3) & ~3);
  float* sWh = sfilt + (size_t)w * KP;
  float* sF = sWh + (size_t)K * M;
  float* sdF = sF + (size_t)tc_cap * KP;
  float* sde = sdF + (size_t)tc_cap * KP;
  float* sdm = sde + ((tc_cap + 3) & ~3);
  float* sdctx = sdm + (size_t)AB_TILE * M;
  float* sred = sdctx + E;

  const int b0 = a.win[0], b1 = a.win[1];
  const int Tw = max(0, b1 - b0);
  const int tc = (Tw + AB_CS - 1) / AB_CS;
  const int t0 = min(Tw, rank * tc), t1 = min(Tw, t0 + tc);
  const int nt = t1 - t0;

  // ---- stage: alpha_{i-1} slice (zero padding relative to the CUT), filters, handler, dctx ----
  for (int i = tid; i < nt + 2 * n + 8; i += AB_NT) {
    const int prel = t0 - n + i;
    salpha[i] = (prel >= 0 && prel < Tw) ? a.w_prev[(long long)b * Tp + b0 + prel] : 0.f;
  }
  for (int i = tid; i < w * KP; i += AB_NT) { const int j = i / KP, k = i % KP; sfilt[i] = k < K ? a.filt[(size_t)k * w + j] : 0.f; }
  for (int i = tid; i < K * M; i += AB_NT) sWh[i] = a.Wh[i];
  for (int i = tid; i < E; i += AB_NT) sdctx[i] = a.dctx[(long long)b * E + i];
  // S = sum_t alpha_i[t] dalpha_i[t] = dctx . ctx_i + sum_t alpha_i[t] carry[t]
  float part = 0.f;
  for (int i = tid; i < E; i += AB_NT) part += a.dctx[(long long)b * E + i] * a.ctx[(long long)b * E + i];
  if (a.dA_in)
    for (int t = tid; t < Tw; t += AB_NT) {
      const long long o = (long long)b * Tp + b0 + t;
      part += a.w_cur[o] * (a.dA_in[o] + a.dA_in[(long long)B * Tp + o]);
    }
  if (a.pen)           // the penalty's gradient of alpha_i joins the carry
    for (int t = tid; t < Tw; t += AB_NT) {
      const long long o = (long long)b * Tp + b0 + t;
      part += a.w_cur[o] * a.pen[o];
    }
  const float S = block_sum_512(part, sred);      // (contains the __syncthreads that publish the staging)

  // ---- de[t] for the owned positions (softmax: alpha_i[t] (dctx . H[t] + carry[t] - S)): one warp per position ----
  for (int t = warp; t < nt; t += AB_NT / 32) {
    const long long pos = b0 + t0 + t;
    const float* hrow = a.H + (pos * B + b) * E;
    float d = 0.f;
    for (int e = lane * 4; e < E; e += 128) {
      const float4 h4 = __ldg(reinterpret_cast<const float4*>(hrow + e));
      const float4 c4 = *reinterpret_cast<const float4*>(sdctx + e);
      d = fmaf(h4.x, c4.x, d); d = fmaf(h4.y, c4.y, d); d = fmaf(h4.z, c4.z, d); d = fmaf(h4.w, c4.w, d);
    }
    d = warp_sum(d);
    if (lane == 0) {
      const long long o = (long long)b * Tp + pos;
      float carry = a.dA_in ? (a.dA_in[o] + a.dA_in[(long long)B * Tp + o]) : 0.f;
      if (a.pen) carry += a.pen[o];
      if constexpr (NORM == LVSR_NORM_SOFTMAX) {
        sde[t] = a.w_cur[o] * (d + carry - S);
      } else if constexpr (NORM == LVSR_NORM_LOGISTIC) {
        sde[t] = a.w_cur[o] * (1.f / (1.f + expf(a.e_cur[o]))) * (d + carry - S);      // 1 - sigma(e) = sigma(-e)
      } else {
        const float e = a.e_cur[o];
        sde[t] = e > 0.f ? (d + carry - S) * (a.w_cur[o] / e) : 0.f;
      }
    }
  }
  // ---- location features of the owned positions: F[t,k] = sum_j alpha_cut[t + n - j] filt[k, j];
  //      a position's taps are split over 4 adjacent lanes ----
  {
    const int seg = (w + 3) / 4;
    for (int base = 0; base < nt * 4; base += AB_NT) {
      const int idx = base + tid, t = idx >> 2, jq = idx & 3;
      float acc[KP];
#pragma unroll
      for (int k = 0; k < KP; ++k) acc[k] = 0.f;
      if (t < nt) {
        const int j0 = jq * seg, j1 = min(w, j0 + seg);
        for (int j = j0; j < j1; ++j) {
          const float av = salpha[t + 2 * n - j];
          const float4* fr = reinterpret_cast<const float4*>(sfilt + (size_t)j * KP);
#pragma unroll
          for (int q = 0; q < KV; ++q) {
            const float4 f = fr[q];
            acc[4 * q] = fmaf(av, f.x, acc[4 * q]); acc[4 * q + 1] = fmaf(av, f.y, acc[4 * q + 1]);
            acc[4 * q + 2] = fmaf(av, f.z, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(av, f.w, acc[4 * q + 3]);
          }
        }
      }
#pragma unroll
      for (int k = 0; k < KP; ++k) {
        acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], 1);
        acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], 2);
      }
      if (t < nt && jq == 0) {
#pragma unroll
        for (int q = 0; q < KV; ++q)
          *reinterpret_cast<float4*>(sF + (size_t)t * KP + 4 * q) = make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
      }
    }
  }
  __syncthreads();

  // ---- main pass over the owned positions, 16 at a time -------------------------------------
  const bool col = tid < M;
  const int m = col ? tid : 0;
  const float qm = a.q[(long long)b * M + m], vm = a.v[m];
  float whc[KP], dWh[KP];
#pragma unroll
  for (int k = 0; k < KP; ++k) { whc[k] = k < K ? sWh[(size_t)k * M + m] : 0.f; dWh[k] = 0.f; }
  float dq = 0.f, dv = 0.f;
  const int MQ = M / 128;                       // float4 groups of a handler row per lane in the dF pass
  for (int tile = 0; tile * AB_TILE < nt; ++tile) {
    const int tb = tile * AB_TILE, tn = min(AB_TILE, nt - tb);
    if (col) {
      float pv[AB_TILE], dpv[AB_TILE];
#pragma unroll
      for (int tl = 0; tl < AB_TILE; ++tl) {
        if (tl < tn) {
          const long long o = ((long long)(b0 + t0 + tb + tl) * B + b) * M + m;
          pv[tl] = __ldg(a.P + o);
          dpv[tl] = a.dP[o];
        }
      }
#pragma unroll
      for (int tl = 0; tl < AB_TILE; ++tl) {
        float dm = 0.f;
        if (tl < tn) {
          const float4* fr4 = reinterpret_cast<const float4*>(sF + (size_t)(tb + tl) * KP);
          float fr[KP];
#pragma unroll
          for (int q = 0; q < KV; ++q) { const float4 f = fr4[q]; fr[4 * q] = f.x; fr[4 * q + 1] = f.y; fr[4 * q + 2] = f.z; fr[4 * q + 3] = f.w; }
          float f = 0.f;
#pragma unroll
          for (int k = 0; k < KP; ++k) f = fmaf(fr[k], whc[k], f);
          const float th = tanhf_acc(pv[tl] + qm + f);
          const float de = sde[tb + tl];
          dm = de * vm * (1.f - th * th);
          a.dP[((long long)(b0 + t0 + tb + tl) * B + b) * M + m] = dpv[tl] + dm;
          dq += dm;
          dv = fmaf(de, th, dv);
#pragma unroll
          for (int k = 0; k < KP; ++k) dWh[k] = fmaf(fr[k], dm, dWh[k]);
        }
        sdm[(size_t)tl * M + m] = dm;
      }
    }
    __syncthreads();
    // dF[t, k] = sum_m dmatch[t, m] Wh[k, m]: warp tl; lane covers m = 4 lane + 128 q (conflict-free float4 rows)
    if (warp < tn) {
      const float4* dmr = reinterpret_cast<const float4*>(sdm + (size_t)warp * M);
      float4 dmv[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) dmv[q] = q < MQ ? dmr[q * 32 + lane] : make_float4(0.f, 0.f, 0.f, 0.f);
      float* out = sdF + (size_t)(tb + warp) * KP;
      for (int k = 0; k < KP; ++k) {
        float s = 0.f;
        if (k < K) {
          const float4* wr = reinterpret_cast<const float4*>(sWh + (size_t)k * M);
#pragma unroll
          for (int q = 0; q < 4; ++q)
            if (q < MQ) {
              const float4 w4 = wr[q * 32 + lane];
              s = fmaf(dmv[q].x, w4.x, s); s = fmaf(dmv[q].y, w4.y, s); s = fmaf(dmv[q].z, w4.z, s); s = fmaf(dmv[q].w, w4.w, s);
            }
          s = warp_sum(s);
        }
        if (lane == 0) out[k] = s;
      }
    }
    __syncthreads();
  }
  // ---- per-step outputs and the running partial sums of this CTA ------------------------------
  if (col) {
    a.dq_part[((long long)rank * B + b) * M + m] = dq;
    a.acc_v[(long long)blockIdx.x * M + m] += dv;
#pragma unroll
    for (int k = 0; k < KP; ++k)
      if (k < K) a.acc_Wh[((long long)blockIdx.x * K + k) * M + m] += dWh[k];
  }
  if constexpr (NORM != LVSR_NORM_SOFTMAX) {
    // energy bias: the owned positions' de, summed by the last warp in a fixed order
    if (warp == AB_NT / 32 - 1) {
      float s = 0.f;
      for (int t = lane; t < nt; t += 32) s += sde[t];
      s = warp_sum(s);
      if (lane == 0) a.acc_b[blockIdx.x] += s;
    }
  }
  // gradient of alpha_{i-1}: dalpha_cut[t'] = sum_j dF[t' - n + j, :] . filt[:, j] over the OWNED t = t' - n + j
  for (int pidx = tid; pidx < Tp; pidx += AB_NT) {
    float acc = 0.f;
    const int tp = pidx - b0;                      // window-relative position of the output
    if (tp >= 0 && tp < Tw && nt > 0) {
      const int jlo = max(0, t0 - tp + n), jhi = min(w - 1, t1 - 1 - tp + n);
      for (int j = jlo; j <= jhi; ++j) {
        const float4* dfr = reinterpret_cast<const float4*>(sdF + (size_t)(tp - n + j - t0) * KP);
        const float4* fj = reinterpret_cast<const float4*>(sfilt + (size_t)j * KP);
#pragma unroll
        for (int q = 0; q < KV; ++q) {
          const float4 d4 = dfr[q], f4 = fj[q];
          acc = fmaf(d4.x, f4.x, acc); acc = fmaf(d4.y, f4.y, acc); acc = fmaf(d4.z, f4.z, acc); acc = fmaf(d4.w, f4.w, acc);
        }
      }
    }
    a.dA_out[((long long)rank * B + b) * Tp + pidx] = acc;
  }
  // dfilt[k, j] += sum_t dF[t, k] alpha_cut[t + n - j]: a tap's positions are split over 2 adjacent lanes
  for (int base = 0; base < 2 * w; base += AB_NT) {
    const int idx = base + tid, j = idx >> 1, th = idx & 1;
    float acc[KP];
#pragma unroll
    for (int k = 0; k < KP; ++k) acc[k] = 0.f;
    if (j < w) {
      const int half = (nt + 1) / 2, ta = th * half, tb2 = min(nt, ta + half);
      for (int t = ta; t < tb2; ++t) {
        const float av = salpha[t + 2 * n - j];
        const float4* dfr = reinterpret_cast<const float4*>(sdF + (size_t)t * KP);
#pragma unroll
        for (int q = 0; q < KV; ++q) {
          const float4 d4 = dfr[q];
          acc[4 * q] = fmaf(av, d4.x, acc[4 * q]); acc[4 * q + 1] = fmaf(av, d4.y, acc[4 * q + 1]);
          acc[4 * q + 2] = fmaf(av, d4.z, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(av, d4.w, acc[4 * q + 3]);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < KP; ++k) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], 1);
    if (j < w && th == 0) {
#pragma unroll
      for (int k = 0; k < KP; ++k)
        if (k < K) a.acc_filt[(long long)blockIdx.x * K * w + (size_t)k * w + j] += acc[k];
    }
  }
}

// Content-only attention (SequenceContentAttention, B/bricks/attention.py:259-414): the same step backward without the
// location term -- no conv recompute, no dF, no handler / filter partials and no gradient into alpha_{i-1} (the weights
// of step i depend on s_{i-1} and the attended sequence only).  Every frame is attended: the window is [0, Tp).
__host__ __device__ inline size_t att_bwd_content_smem_floats(int E, int tc_cap) {
  return (size_t)((tc_cap + 3) & ~3) + E + 64 + 16;     // sde | sdctx | block reductions
}

__global__ void __launch_bounds__(AB_NT, 1) att_bwd_content_kernel(AttBwdArgs a, int tc_cap) {
  extern __shared__ __align__(16) float smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.x / AB_CS, rank = blockIdx.x % AB_CS;
  const int M = a.M, E = a.E, Tp = a.Tp, B = a.B;
  float* sde = smem;
  float* sdctx = sde + ((tc_cap + 3) & ~3);
  float* sred = sdctx + E;
  const int tc = (Tp + AB_CS - 1) / AB_CS;
  const int t0 = min(Tp, rank * tc), t1 = min(Tp, t0 + tc);
  const int nt = t1 - t0;

  for (int i = tid; i < E; i += AB_NT) sdctx[i] = a.dctx[(long long)b * E + i];
  // S = sum_t alpha_i[t] dalpha_i[t] = dctx . ctx_i
  float part = 0.f;
  for (int i = tid; i < E; i += AB_NT) part += a.dctx[(long long)b * E + i] * a.ctx[(long long)b * E + i];
  if (a.pen)           // + sum_t alpha_i[t] pen[t]: the penalty's gradient of alpha_i
    for (int t = tid; t < Tp; t += AB_NT) part += a.w_cur[(long long)b * Tp + t] * a.pen[(long long)b * Tp + t];
  const float S = block_sum_512(part, sred);      // (contains the __syncthreads that publish the staging)

  // ---- de[t] = alpha_i[t] (dctx . H[t] (+ pen[t]) - S) for the owned positions: one warp per position ----
  for (int t = warp; t < nt; t += AB_NT / 32) {
    const long long pos = t0 + t;
    const float* hrow = a.H + (pos * B + b) * E;
    float d = 0.f;
    for (int e = lane * 4; e < E; e += 128) {
      const float4 h4 = __ldg(reinterpret_cast<const float4*>(hrow + e));
      const float4 c4 = *reinterpret_cast<const float4*>(sdctx + e);
      d = fmaf(h4.x, c4.x, d); d = fmaf(h4.y, c4.y, d); d = fmaf(h4.z, c4.z, d); d = fmaf(h4.w, c4.w, d);
    }
    d = warp_sum(d);
    if (lane == 0) {
      const long long o = (long long)b * Tp + pos;
      sde[t] = a.pen ? a.w_cur[o] * (d + a.pen[o] - S) : a.w_cur[o] * (d - S);
    }
  }
  __syncthreads();

  // ---- one thread per matcher column, 16 positions of P and dP in flight ----
  if (tid >= M) return;
  const int m = tid;
  const float qm = a.q[(long long)b * M + m], vm = a.v[m];
  float dq = 0.f, dv = 0.f;
  for (int tb = 0; tb < nt; tb += AB_TILE) {
    const int tn = min(AB_TILE, nt - tb);
    float pv[AB_TILE], dpv[AB_TILE];
#pragma unroll
    for (int tl = 0; tl < AB_TILE; ++tl) {
      if (tl < tn) {
        const long long o = ((long long)(t0 + tb + tl) * B + b) * M + m;
        pv[tl] = __ldg(a.P + o);
        dpv[tl] = a.dP[o];
      }
    }
#pragma unroll
    for (int tl = 0; tl < AB_TILE; ++tl) {
      if (tl < tn) {
        const float th = tanhf_acc(pv[tl] + qm);
        const float de = sde[tb + tl];
        const float dm = de * vm * (1.f - th * th);
        a.dP[((long long)(t0 + tb + tl) * B + b) * M + m] = dpv[tl] + dm;
        dq += dm;
        dv = fmaf(de, th, dv);
      }
    }
  }
  a.dq_part[((long long)rank * B + b) * M + m] = dq;
  a.acc_v[(long long)blockIdx.x * M + m] += dv;
}

// out[i] = sum over the CTAs' partials (fixed order)
__global__ void reduce_partials_kernel(const float* part, int nparts, long long n, float* out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int p = 0; p < nparts; ++p) s += part[(long long)p * n + i];
    out[i] = s;
  }
}

// sum of all elements -> out[0] (single CTA; the cost scalar)
__global__ void __launch_bounds__(1024) sum_all_kernel(const float* x, long long n, float* out, float scale) {
  __shared__ float red[32];
  float s = 0.f;
  for (long long i = threadIdx.x; i < n; i += 1024) s += x[i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = red[threadIdx.x];
    v = warp_sum(v);
    if (threadIdx.x == 0) out[0] = v * scale;
  }
}

// ------------------------------------------------------------------------------------------
// Step rules (lvsr/main.py:480-519): StepClipping -> Momentum -> AdaDelta -> Restrict(VariableClipping(axis=0),
// WEIGHT) -> RemoveNotFinite(0.0) -> BurnIn, then parameter -= step.  All on the flat layout.
// ------------------------------------------------------------------------------------------
struct ParamDesc { long long offset; int rows, cols; int is_weight; };

// partial sums of squares of g * gscale, one per CTA (deterministic two-level reduction)
__global__ void __launch_bounds__(256) sqnorm_partial_kernel(const float* g, long long n, float* part) {
  __shared__ float red[8];
  float s = 0.f;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) s = fmaf(g[i], g[i], s);
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
    for (int q = 0; q < 8; ++q) v += red[q];
    part[blockIdx.x] = v;
  }
}
// Adaptive clipping (lvsr/extensions.py:64-91 as lvsr/main.py:616-619 installs it; lvsr_train_set_adaptive_clipping):
// device doubles.  CLIP_THR is the threshold of the step being applied, CLIP_NEXT the one the next step will use.
enum { CLIP_MU = 0, CLIP_MU2 = 1, CLIP_N = 2, CLIP_THR = 3, CLIP_NEXT = 4, CLIP_THR0 = 5, CLIP_DECAY = 6, CLIP_BURNIN = 7,
       CLIP_WORDS = 8 };

// AdaptiveClipping.after_batch for the batch whose gradient norm is `norm`, in float64.  A zero norm (math.log(0) raises
// in the reference) leaves the moments as they were; the count still advances, as iterations_done does.
__device__ inline void adaptive_clip_update(double* c, double norm) {
  c[CLIP_THR] = c[CLIP_NEXT];
  const double d = c[CLIP_DECAY], thr0 = c[CLIP_THR0], burnin = c[CLIP_BURNIN];
  const double n = c[CLIP_N] + 1.0;
  c[CLIP_N] = n;
  if (norm != 0.0) {
    const double L = log(norm);
    c[CLIP_MU] = d * c[CLIP_MU] + (1.0 - d) * L;
    c[CLIP_MU2] = d * c[CLIP_MU2] + (1.0 - d) * L * L;
  }
  const double mu = c[CLIP_MU], var = c[CLIP_MU2] - mu * mu;
  const double sigma = sqrt(var < 0.0 ? 0.0 : var);          // rounding below 0 only; a NaN passes through
  const double conf = fmin(burnin, n) / burnin;
  const double thr = conf * exp(mu + sigma) + (1.0 - conf) * thr0;
  const double cap = 5.0 * thr0;
  c[CLIP_NEXT] = cap < thr ? cap : thr;                       // Python's min(thr, cap): a NaN threshold stays NaN
}

// clip: adaptive clipping state or nullptr (off)
__global__ void sqnorm_final_kernel(const float* part, int nparts, float gscale, float* norm_out, double* clip) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < nparts; ++i) s += (double)part[i];
    const float norm = (float)(sqrt(s) * (double)gscale);
    norm_out[0] = norm;
    if (clip) adaptive_clip_update(clip, (double)norm);
  }
}

struct StepArgs {
  float* grads;              // in: summed gradients; out: the step
  const float* params;
  float* velocity; float* ms_step; float* ms_dx;
  const float* norm;         // [1] L2 norm of gscale * grads
  long long n;
  float gscale;              // 1 / global batch size
  float decay;               // weight decay coefficient (lvsr/main.py:419-421): grad += 2 decay W on WEIGHTs
  float threshold;           // StepClipping (0 = off)
  int use_momentum; float learning_rate, momentum;
  int use_adadelta; float decay_rate, epsilon;
  const unsigned char* is_weight_map;   // per element or nullptr
  const double* clip;        // adaptive clipping state or nullptr: the threshold is clip[CLIP_THR], not `threshold`
};
__global__ void step_rules_kernel(StepArgs a) {
  const float norm = a.norm[0];
  float mult;
  if (a.clip) {              // StepClipping with its shared float32 threshold: switch(norm < thr, 1, thr / norm)
    const float thr = (float)a.clip[CLIP_THR];
    mult = norm < thr ? 1.f : thr / norm;
  } else {
    mult = (a.threshold > 0.f && !(norm < a.threshold)) ? a.threshold / norm : 1.f;
  }
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < a.n; i += (long long)gridDim.x * blockDim.x) {
    float s = a.grads[i] * a.gscale * mult;
    if (a.use_momentum) {
      s = a.momentum * a.velocity[i] + a.learning_rate * s;
      a.velocity[i] = s;
    }
    if (a.use_adadelta) {
      const float ms = a.decay_rate * a.ms_step[i] + (1.f - a.decay_rate) * s * s;
      const float dx = sqrtf(a.ms_dx[i] + a.epsilon) / sqrtf(ms + a.epsilon) * s;
      a.ms_step[i] = ms;
      a.ms_dx[i] = a.decay_rate * a.ms_dx[i] + (1.f - a.decay_rate) * dx * dx;
      s = dx;
    }
    a.grads[i] = s;
  }
}
// weight decay is part of the gradient: applied BEFORE the norm (grads += 2 decay W / gscale so that the later
// multiplication by gscale leaves 2 decay W)
__global__ void add_decay_kernel(float* grads, const float* params, const ParamDesc* desc, int nparams, float coef) {
  const ParamDesc d = desc[blockIdx.y];
  if (!d.is_weight) return;
  const long long cnt = (long long)d.rows * d.cols;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < cnt; i += (long long)gridDim.x * blockDim.x)
    grads[d.offset + i] += coef * params[d.offset + i];
}

// VariableClipping(max_norm, axis=0) on WEIGHT parameters: per column c, if || p[:, c] - s[:, c] || > thr:
// s = p - thr / norm * (p - s).   One warp per column.
__global__ void __launch_bounds__(256) max_norm_kernel(float* step, const float* params, const ParamDesc* desc, float thr) {
  const ParamDesc d = desc[blockIdx.y];
  if (!d.is_weight) return;
  const int lane = threadIdx.x & 31;
  for (int c = blockIdx.x * 8 + (threadIdx.x >> 5); c < d.cols; c += gridDim.x * 8) {
    float ss = 0.f;
    for (int r = lane; r < d.rows; r += 32) {
      const long long o = d.offset + (long long)r * d.cols + c;
      const float nv = params[o] - step[o];
      ss = fmaf(nv, nv, ss);
    }
    ss = warp_sum(ss);
    const float norm = sqrtf(ss);
    if (norm > thr) {
      const float f = thr / norm;
      for (int r = lane; r < d.rows; r += 32) {
        const long long o = d.offset + (long long)r * d.cols + c;
        step[o] = params[o] - f * (params[o] - step[o]);
      }
    }
  }
}
// RemoveNotFinite(0.0) + BurnIn + the update of one parameter by one CTA.
__device__ __forceinline__ void apply_update_param(float* params, const float* step, const ParamDesc d, float burn_mult) {
  const long long cnt = (long long)d.rows * d.cols;
  __shared__ float red[8];
  __shared__ int bad;
  float s = 0.f;
  for (long long i = threadIdx.x; i < cnt; i += 256) s += step[d.offset + i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
    for (int q = 0; q < 8; ++q) v += red[q];
    bad = (isnan(v) || isinf(v)) ? 1 : 0;
  }
  __syncthreads();
  for (long long i = threadIdx.x; i < cnt; i += 256) {
    const long long o = d.offset + i;
    // RemoveNotFinite(scaler = 0.0): step = (1 - 0) * parameter  ->  the parameter becomes 0 (B/algorithms/__init__.py:855-861)
    const float st = bad ? params[o] : step[o];
    params[o] = params[o] - st * burn_mult;
  }
}
__global__ void __launch_bounds__(256) apply_update_kernel(float* params, const float* step, const ParamDesc* desc, float burn_mult) {
  apply_update_param(params, step, desc[blockIdx.x], burn_mult);
}
// Adaptive noise: the updates of the means (CTAs [0, nparams)) and of their log-variances (CTAs [nparams, 2 nparams))
// in one grid, so that the CTA of a large log-variance runs beside, not after, the CTA of its large mean.
__global__ void __launch_bounds__(256) apply_update_pair_kernel(float* params, const float* step, float* params2,
                                                                const float* step2, const ParamDesc* desc, int nparams,
                                                                float burn_mult) {
  const bool second = (int)blockIdx.x >= nparams;
  apply_update_param(second ? params2 : params, second ? step2 : step, desc[blockIdx.x - (second ? nparams : 0)], burn_mult);
}

}  // namespace train
}  // namespace lvsr
