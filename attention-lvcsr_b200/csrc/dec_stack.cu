// Upper layer of the stacked decoder (dec_stack 2): RecurrentStack([GRU transition_0, GRU transition_1],
// skip_connections=True) as lvsr/bricks/recognizer.py:250-259 builds it.  Layer 0 is the single-layer decoder's step
// (api.cu: transition); this file is layer 1's step, whose inputs are the sum of the generator's feedback fork
// (inputs#1, with bias), the distributed glimpses (distribute/fork_*#1) and the stack's bias-free fork_1 of layer 0's
// new state (libs/blocks/blocks/bricks/recurrent.py:925-950).
//
// Same tiling as decoder.cu's dense_kernel -- a CTA owns 8 output columns for a block of 64 rows, its 8 warps split
// the contraction and meet in shared memory, the GRU non-linearities are fused into the epilogue -- with one row
// stride per operand, so the layer reads and writes the upper half of the wide state rows [s0 | s1] in place.
#include "kernels.h"
#include "lvsr_b200.h"

namespace lvsr {

namespace {

constexpr int SR = 64;   // rows per CTA
constexpr int SN = 8;    // columns per CTA
enum { STACK_GATES = 0, STACK_CAND = 1 };

struct Operand { const float* X; int K, ldx; const float* W; int ldw, ncols; };   // X[R, K] . W[K, :ncols]

// out[R, N] = epilogue(sum of the operands + add[arow[r]])
struct StackDense {
  Operand op[3];
  int nop;
  const float* add; const long long* arow; long long add_rows; int ld_add;
  int R, N, mode, C;
  const float* s; int ld_s;         // layer 1's current state
  float *z, *hr, *ai;               // STACK_GATES: cols [0,C) -> z, [C,2C) -> hr = s * r, [2C,3C) -> ai
  const float* rmask;               // STACK_CAND: c = tanh(acc + ai), s' = c z + s (1 - z), row-mask blend
  float* out; int ld_out;
};

__global__ void __launch_bounds__(256) stack_dense_kernel(StackDense a) {
  __shared__ __align__(16) float red[8][SR * SN];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n0 = blockIdx.x * SN, r0 = blockIdx.y * SR;
  const int rg = lane >> 1, cgp = lane & 1;
  const int c0 = n0 + cgp * 4;                 // first of 4 columns of this lane
  const int rbase = r0 + rg * 4;               // first of 4 rows of this lane

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int o = 0; o < a.nop; ++o) {
    const Operand p = a.op[o];
    if (c0 >= p.ncols) continue;
    const int kq = (p.K / 4 + 7) / 8;          // float4 groups per warp
    const int k_lo = min(p.K, warp * kq * 4), k_hi = min(p.K, k_lo + kq * 4);
    const float* xr[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) xr[i] = p.X + (long long)min(rbase + i, a.R - 1) * p.ldx;
    for (int k = k_lo; k + 4 <= k_hi; k += 4) {
      float4 xv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) xv[i] = *reinterpret_cast<const float4*>(xr[i] + k);
      float4 wv[4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wv[kk] = __ldg(reinterpret_cast<const float4*>(p.W + (long long)(k + kk) * p.ldw + c0));
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
  }

#pragma unroll
  for (int i = 0; i < 4; ++i)
    *reinterpret_cast<float4*>(&red[warp][(rg * 4 + i) * SN + cgp * 4]) =
        make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
  __syncthreads();

  for (int o = tid; o < SR * SN; o += 256) {
    const int rl = o / SN, cl = o % SN;
    const int r = r0 + rl, c = n0 + cl;
    if (r >= a.R || c >= a.N) continue;
    float v = 0.f;
#pragma unroll
    for (int wq = 0; wq < 8; ++wq) v += red[wq][o];
    long long ar = a.arow ? a.arow[r] : (long long)r;
    if (a.arow) ar = ar < 0 ? 0 : (ar > a.add_rows - 1 ? a.add_rows - 1 : ar);
    v += a.add[ar * a.ld_add + c];
    const int C = a.C;
    if (a.mode == STACK_GATES) {
      if (c < C) {
        a.z[(long long)r * C + c] = sigmoidf_acc(v);
      } else if (c < 2 * C) {
        const int u = c - C;
        a.hr[(long long)r * C + u] = a.s[(long long)r * a.ld_s + u] * sigmoidf_acc(v);
      } else {
        a.ai[(long long)r * C + (c - 2 * C)] = v;
      }
    } else {
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

int launch(const StackDense& d, cudaStream_t stream) {
  for (int o = 0; o < d.nop; ++o)
    LVSR_CHECK(d.op[o].K % 4 == 0 && d.op[o].ldx % 4 == 0 && d.op[o].ldw % 4 == 0 && d.op[o].ncols % 4 == 0,
               "stack_upper_step: dimensions and strides must be multiples of 4");
  dim3 grid(ceil_div(d.N, SN), ceil_div(d.R, SR));
  stack_dense_kernel<<<grid, 256, 0, stream>>>(d);
  LVSR_LAUNCH_CHECK();
  return 0;
}

}  // namespace

int stack_upper_step(const StackUpperArgs& a, cudaStream_t stream) {
  ProfScope prof("dense", stream);
  if (a.R <= 0) return 0;
  const int C = a.C;
  StackDense g = {};
  g.op[0] = {a.ctx, a.E, a.E, a.Wd, 3 * C, 3 * C};
  g.op[1] = {a.s0n, C, a.ld_s0n, a.F, 3 * C, 3 * C};
  g.op[2] = {a.s1, C, a.ld_s1, a.U, 2 * C, 2 * C};       // state_to_gates feeds the gate columns only
  g.nop = 3;
  g.add = a.FF; g.arow = a.outputs; g.add_rows = a.ff_rows; g.ld_add = 3 * C;
  g.R = a.R; g.N = 3 * C; g.mode = STACK_GATES; g.C = C;
  g.s = a.s1; g.ld_s = a.ld_s1; g.z = a.z; g.hr = a.hr; g.ai = a.ai;
  if (int rc = launch(g, stream)) return rc;
  StackDense k = {};
  k.op[0] = {a.hr, C, C, a.W, C, C};
  k.nop = 1;
  k.add = a.ai; k.arow = nullptr; k.ld_add = C;
  k.R = a.R; k.N = C; k.mode = STACK_CAND; k.C = C;
  k.s = a.s1; k.ld_s = a.ld_s1; k.z = a.z; k.rmask = a.rmask; k.out = a.out; k.ld_out = a.ld_out;
  return launch(k, stream);
}

}  // namespace lvsr
