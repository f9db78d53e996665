// Dense projections of the path: C[M,N] (+)= A[M,K] . W[K,N] + bias.
//
// Replaces every whole-sequence tensor.dot of the reference graph:
//   Fork(Linear) of RecurrentWithFork  (lvsr/bricks/__init__.py:39-43, B/bricks/simple.py:73-76)
//   attention.preprocess               (lvsr/bricks/attention.py:228-230)
//   Readout merge                      (B/bricks/sequence_generators.py:614-619)
//   post_merge MLP hidden layers       (lvsr/bricks/recognizer.py:305-320; act(. + b) in the epilogue)
//
// fp32 FFMA tiles (128x128x8, 8x8 per thread, double-buffered shared memory): the
// 1e-4 parity gate against the float64 oracle rules out single-pass bf16/tf32 here.
// A rows may be a strided view of a [T,B,K] tensor (the encoder's x[::k]).
#include "kernels.h"

namespace lvsr {

namespace {

constexpr int BM = 128, BN = 128, BK = 8;
constexpr int APAD = 4;

// the readout hidden layers' activations (readout_act in decoder.cu): Rectifier as fmaxf, Tanh
template <int ACT>
__device__ __forceinline__ float epilogue_act(float v) {
  if (ACT == LVSR_ACT_RELU) return fmaxf(v, 0.f);
  if (ACT == LVSR_ACT_TANH) return tanhf(v);
  return v;
}

// ACT: GemmArgs::act as a template argument (LVSR_ACT_IDENTITY: no activation)
template <bool VEC, int ACT>
__global__ void __launch_bounds__(256)
gemm_kernel(GemmArgs g) {
  __shared__ __align__(16) float As[2][BK][BM + APAD];
  __shared__ __align__(16) float Bs[2][BK][BN];

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

  // A loader: one float4 (4 consecutive k) of one row per thread
  const int a_row = tid >> 1, a_kq = (tid & 1) * 4;
  const int gr = m0 + a_row;
  const float* a_ptr = nullptr;
  if (gr < g.M) {
    a_ptr = g.A + (long long)(gr / g.rows_per_block) * g.block_stride +
            (long long)(gr % g.rows_per_block) * g.lda;
  }
  // B loader: one float4 (4 consecutive n) of one k per thread
  const int b_k = tid >> 5, b_n = (tid & 31) * 4;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 ra, rb;
  auto load_tiles = [&](int k0) {
    ra = make_float4(0.f, 0.f, 0.f, 0.f);
    rb = make_float4(0.f, 0.f, 0.f, 0.f);
    const int ka = k0 + a_kq;
    if (a_ptr != nullptr) {
      if (VEC) {
        if (ka < g.K) ra = *reinterpret_cast<const float4*>(a_ptr + ka);
      } else {
        if (ka + 0 < g.K) ra.x = a_ptr[ka + 0];
        if (ka + 1 < g.K) ra.y = a_ptr[ka + 1];
        if (ka + 2 < g.K) ra.z = a_ptr[ka + 2];
        if (ka + 3 < g.K) ra.w = a_ptr[ka + 3];
      }
    }
    const int kb = k0 + b_k;
    const int nb = n0 + b_n;
    if (kb < g.K) {
      const float* wp = g.W + (long long)kb * g.ldw + nb;
      if (VEC) {
        if (nb < g.N) rb = *reinterpret_cast<const float4*>(wp);
      } else {
        if (nb + 0 < g.N) rb.x = wp[0];
        if (nb + 1 < g.N) rb.y = wp[1];
        if (nb + 2 < g.N) rb.z = wp[2];
        if (nb + 3 < g.N) rb.w = wp[3];
      }
    }
  };
  auto store_tiles = [&](int buf) {
    As[buf][a_kq + 0][a_row] = ra.x;
    As[buf][a_kq + 1][a_row] = ra.y;
    As[buf][a_kq + 2][a_row] = ra.z;
    As[buf][a_kq + 3][a_row] = ra.w;
    *reinterpret_cast<float4*>(&Bs[buf][b_k][b_n]) = rb;
  };

  const int nk = (g.K + BK - 1) / BK;
  load_tiles(0);
  store_tiles(0);
  __syncthreads();

  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_tiles((kt + 1) * BK);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_tiles(buf ^ 1);
      __syncthreads();
    }
  }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (r >= g.M) continue;
    float* crow = g.C + (long long)r * g.ldc;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int c = n0 + jh * 64 + tx * 4;
      if (c >= g.N) continue;
      float v[4] = {acc[i][jh * 4 + 0], acc[i][jh * 4 + 1], acc[i][jh * 4 + 2], acc[i][jh * 4 + 3]};
      if (VEC) {
        if (g.bias) {
          const float4 bb = *reinterpret_cast<const float4*>(g.bias + c);
          v[0] += bb.x; v[1] += bb.y; v[2] += bb.z; v[3] += bb.w;
        }
        float4* cp = reinterpret_cast<float4*>(crow + c);
        if (g.accumulate) {
          const float4 o = *cp;
          v[0] += o.x; v[1] += o.y; v[2] += o.z; v[3] += o.w;
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) v[q] = epilogue_act<ACT>(v[q]);
        *cp = make_float4(v[0], v[1], v[2], v[3]);
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          if (c + q < g.N) {
            float o = v[q] + (g.bias ? g.bias[c + q] : 0.f);
            if (g.accumulate) o += crow[c + q];
            crow[c + q] = epilogue_act<ACT>(o);
          }
        }
      }
    }
  }
}

template <bool VEC>
void launch_gemm(const GemmArgs& g, dim3 grid, cudaStream_t stream) {
  if (g.act == LVSR_ACT_RELU) gemm_kernel<VEC, LVSR_ACT_RELU><<<grid, 256, 0, stream>>>(g);
  else if (g.act == LVSR_ACT_TANH) gemm_kernel<VEC, LVSR_ACT_TANH><<<grid, 256, 0, stream>>>(g);
  else gemm_kernel<VEC, LVSR_ACT_IDENTITY><<<grid, 256, 0, stream>>>(g);
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace

int gemm_bias(const GemmArgs& g, cudaStream_t stream) {
  ProfScope prof("gemm", stream);
  if (g.M <= 0 || g.N <= 0) return 0;
  LVSR_CHECK(g.K > 0 && g.rows_per_block > 0, "gemm: bad shape");
  const bool vec = (g.K % 4 == 0) && (g.lda % 4 == 0) && (g.block_stride % 4 == 0) &&
                   (g.N % 4 == 0) && (g.ldw % 4 == 0) && (g.ldc % 4 == 0) && aligned16(g.A) &&
                   aligned16(g.W) && aligned16(g.C) && (g.bias == nullptr || aligned16(g.bias));
  dim3 grid(ceil_div(g.N, BN), ceil_div(g.M, BM));
  if (vec)
    launch_gemm<true>(g, grid, stream);
  else
    launch_gemm<false>(g, grid, stream);
  LVSR_LAUNCH_CHECK();
  return 0;
}

}  // namespace lvsr
