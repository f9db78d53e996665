// Tensor-core path for the dense projections: C[M,N] = A[M,K] . W[K,N] + bias on the Hopper
// warpgroup tensor cores (wgmma.mma_async, fp32 accumulators in registers, operands staged by TMA into 128B-swizzled
// shared memory).
//
// Replaces the whole-sequence tensor.dot of Fork(Linear) in RecurrentWithFork
// (lvsr/bricks/__init__.py:39-43) and attention.preprocess (lvsr/bricks/attention.py:228-230):
// the only genuinely dense contractions of the path (SURVEY.md 8a-a2: 260 GFLOP per batch).
//
// Precision: the 1e-4 gate against the float64 oracle rules out a single pass of tf32 or fp16 (2^-11 per product).
// Every operand is split into two parts and three products are accumulated in fp32, small terms first
// (lo.hi + hi.lo + hi.hi; the dropped lo.lo term is 2^-22).  One kernel template, two operand kinds:
//  * tf32 (F16 = false): x = hi + lo EXACTLY, hi = x with the low 13 mantissa bits cleared, lo = tf32(x - hi).  Any K
//    (zero-padded to a multiple of 32); the backward products and contractions that are not a multiple of 64.
//  * fp16 (F16 = true): every row of A and every column of W is first scaled by a power of two 2^e that puts its
//    largest magnitude into [2^13, 2^14), then x 2^e = head + tail with head = fp16(x 2^e), tail = fp16(x 2^e - head).
//    The representation error is 2^-22 of |x 2^e|, or 2^-25 absolute once the tail falls into the fp16 subnormals (2^-38
//    of the row's or column's largest value).  The epilogue unscales exactly: C = ldexp(acc, -(e_row + e_col)) + bias.
//    Half the operand bytes and twice the tf32 rate: K a multiple of 64, the forward projections.
// A is split by one streaming pass per GEMM (split_tf32_kernel / split_pad_tf32_kernel, split_rows_f16_kernel); W once
// per lvsr_model_finalize, kept K-major ([N, K]) so both operands use the K-major SWIZZLE_128B canonical layout (wgmma
// reads tf32 operands from shared memory only in K-major form).
//
// Kernel shape: 128 x 128 output tiles, one 128-byte swizzle row per k-block (32 tf32 or 64 fp16 values),
// 3-stage TMA -> wgmma mbarrier pipeline (4 operand tiles = 64 KB per stage), one persistent CTA per SM, three warpgroups:
// warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = consumers, each owning 64 rows of the
// tile (wgmma m64n128k8 / m64n128k16 into registers, then bias add and stores straight from the accumulators).
// On an H100 a 128 x 256 tile (2 stages, 128 accumulators per thread) measured 7 % slower for the
// projections of the metric configuration than this shape (tf32 operands).
#include <cuda.h>
#include <cuda_fp16.h>
#include <limits.h>

#include <algorithm>

#include "kernels.h"

namespace lvsr {

namespace {

constexpr int TC_BM = 128, TC_BN = 128, TC_BK = 32;      // TC_BN: the granularity N must be a multiple of
constexpr int TC_BK_F16 = 64;                            // fp16 values per 128-byte row: the k-block of the fp16 kind
constexpr int TC_THREADS = 384;                          // producer warpgroup + two consumer warpgroups
constexpr int TC_STAGES = 3;
constexpr uint32_t TC_TILE_BYTES = TC_BM * 128;                            // 16 KB: one 128-row operand tile
constexpr uint32_t TC_STAGE_BYTES = 4 * TC_TILE_BYTES;                     // A_hi, A_lo, B_hi, B_lo (heads and tails)
constexpr size_t TC_SMEM = (size_t)TC_STAGES * TC_STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void bar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void bar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void bar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  unsigned long long spins = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    if (ok) break;
    if (++spins > (1ull << 24)) __trap();   // a broken pipeline must fail the launch, not hang the GPU
  }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int x, int y, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];\n" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(bar)
      : "memory");
}

// ---- wgmma ---------------------------------------------------------------------------------------------------------
// K-major, SWIZZLE_128B canonical layout: rows are 128 B, 8-row groups are 1024 B apart (sm_90 shared-memory matrix
// descriptor: start address, leading byte offset (unused for swizzled K-major), stride byte offset, layout type 1 =
// 128-byte swizzle).  One k-step (8 tf32 or 16 fp16 values = 32 bytes) further along a row is start address + 2.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);          // start address, 16 B units
  d |= (uint64_t)1 << 16;                          // leading byte offset
  d |= (uint64_t)(1024 >> 4) << 32;                // stride byte offset between 8-row groups
  d |= (uint64_t)1 << 62;                          // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// keeps the compiler from touching accumulators across an asynchronous wgmma (reads before the wait, say)
template <int N>
__device__ __forceinline__ void acc_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define LVSR_ACC8(d, i) \
  "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define LVSR_ACC64 "{"                                                                        \
  "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                    \
  "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "          \
  "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "          \
  "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
// d[64] (+)= A (64 x k, K-major) . B (128 x k, K-major)^T: k = 8 tf32 or 16 fp16 values, 32 bytes of each row
template <bool F16>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  if constexpr (F16) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " LVSR_ACC64 ", %64, %65, p, 1, 1, 0, 0;\n\t}\n"
        : LVSR_ACC8(d, 0), LVSR_ACC8(d, 8), LVSR_ACC8(d, 16), LVSR_ACC8(d, 24),
          LVSR_ACC8(d, 32), LVSR_ACC8(d, 40), LVSR_ACC8(d, 48), LVSR_ACC8(d, 56)
        : "l"(desc_a), "l"(desc_b), "r"(scale_d));
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " LVSR_ACC64 ", %64, %65, p, 1, 1;\n\t}\n"
        : LVSR_ACC8(d, 0), LVSR_ACC8(d, 8), LVSR_ACC8(d, 16), LVSR_ACC8(d, 24),
          LVSR_ACC8(d, 32), LVSR_ACC8(d, 40), LVSR_ACC8(d, 48), LVSR_ACC8(d, 56)
        : "l"(desc_a), "l"(desc_b), "r"(scale_d));
  }
}
#undef LVSR_ACC64
#undef LVSR_ACC8

struct TcGemmParams {
  float* C;
  const float* bias;
  const int* ea;               // fp16 operands: exponent of every row of A [M] and column of B [N] (the scaling 2^e)
  const int* eb;
  int M, N, K, ldc;
  int tiles_n, tiles_m, tiles; // output tiles along N and M, and in all (times the splits)
  int kb_per_split;            // K blocks of one split (split-K: partial products, summed by the caller)
  long long c_split_stride;    // elements between the partial outputs of consecutive splits
};

// x 2^-e, exactly unless the result leaves the normal fp32 range: one multiply by a power of two where 2^-e is a normal
// float, ldexpf beyond
__device__ __forceinline__ float unscale(float x, int e) {
  return (unsigned)(e + 126) <= 252u ? x * __uint_as_float((uint32_t)(127 - e) << 23) : ldexpf(x, -e);
}

// TMA producer, one thread: the k-blocks [kb0, kb0 + nkb) of output tile (m0, n0) into the ring of stages.  `it` counts
// the k-blocks this CTA has passed through the ring.
template <int BK>
__device__ __forceinline__ void load_tile(const CUtensorMap* map_a_hi, const CUtensorMap* map_a_lo,
                                          const CUtensorMap* map_b_hi, const CUtensorMap* map_b_lo, uint8_t* tiles,
                                          unsigned long long* bars, int m0, int n0, int kb0, int nkb, uint32_t& it) {
  for (int kb = 0; kb < nkb; ++kb, ++it) {
    const uint32_t s = it % TC_STAGES;
    const uint32_t ph = (it / TC_STAGES) & 1u;
    bar_wait(smem_addr(&bars[TC_STAGES + s]), ph ^ 1u);       // slot free (first round passes immediately)
    const uint32_t full = smem_addr(&bars[s]);
    bar_expect_tx(full, TC_STAGE_BYTES);
    const uint32_t base = smem_addr(tiles + (size_t)s * TC_STAGE_BYTES);
    tma_load_2d(base + 0 * TC_TILE_BYTES, map_a_hi, (kb0 + kb) * BK, m0, full);
    tma_load_2d(base + 1 * TC_TILE_BYTES, map_a_lo, (kb0 + kb) * BK, m0, full);
    tma_load_2d(base + 2 * TC_TILE_BYTES, map_b_hi, (kb0 + kb) * BK, n0, full);
    tma_load_2d(base + 3 * TC_TILE_BYTES, map_b_lo, (kb0 + kb) * BK, n0, full);
  }
}

// Consumer warpgroup wg - 1 (rows [64 (wg - 1), +64) of the tile), thread t: the products of one output tile (N tiles
// fastest, then M tiles, then splits) and its epilogue.  LDG_EA: the row exponents were written before this launch and
// may come through the read-only cache; the streamed kernel writes them while it runs and reads them from L2.
template <bool F16, bool LDG_EA>
__device__ __forceinline__ void mma_store_tile(const TcGemmParams& p, uint8_t* tiles, unsigned long long* bars, int tile,
                                               int wg, int t, uint32_t& it) {
  constexpr int NACC = TC_BN / 2;                       // accumulators per consumer thread (m64 x 128 over 128 threads)
  constexpr int BK = F16 ? TC_BK_F16 : TC_BK;           // values per 128-byte row
  const int total_kb = p.K / BK;
  const uint32_t a_off = (uint32_t)(wg - 1) * 64 * 128;          // 64 rows of 128 bytes into each A tile
  const int warp = t >> 5, lane = t & 31;
  {
    const int n0 = (tile % p.tiles_n) * TC_BN, m0 = (tile / p.tiles_n % p.tiles_m) * TC_BM;
    const int split = tile / (p.tiles_n * p.tiles_m);
    const int nkb = min(p.kb_per_split, total_kb - split * p.kb_per_split);
    float acc[NACC];
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < nkb; ++kb, ++it) {
      const uint32_t s = it % TC_STAGES;
      bar_wait(smem_addr(&bars[s]), (it / TC_STAGES) & 1u);
      const uint32_t base = smem_addr(tiles + (size_t)s * TC_STAGE_BYTES);
      const uint64_t da_hi = make_smem_desc(base + 0 * TC_TILE_BYTES + a_off), da_lo = make_smem_desc(base + 1 * TC_TILE_BYTES + a_off);
      const uint64_t db_hi = make_smem_desc(base + 2 * TC_TILE_BYTES), db_lo = make_smem_desc(base + 3 * TC_TILE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {                      // 4 k-steps of 32 bytes per 128-byte row
        const uint64_t adv = (uint64_t)(k * 2);
        wgmma_n128<F16>(acc, da_lo + adv, db_hi + adv, 1u);     // small terms first
        wgmma_n128<F16>(acc, da_hi + adv, db_lo + adv, 1u);
        wgmma_n128<F16>(acc, da_hi + adv, db_hi + adv, 1u);
      }
      wgmma_commit();
      // the products of the previous k-block have retired: its slot goes back to the producer
      wgmma_wait<1>();
      acc_fence(acc);
      if (kb > 0 && t == 0) bar_arrive(smem_addr(&bars[TC_STAGES + (it - 1) % TC_STAGES]));
    }
    wgmma_wait<0>();
    acc_fence(acc);
    if (t == 0) bar_arrive(smem_addr(&bars[TC_STAGES + (it - 1) % TC_STAGES]));   // the tile's last slot

    // ===== epilogue: accumulator fragment -> global (+bias).  Register 4j + {0,1}: row 16 warp + lane / 4, columns
    // 8j + 2 (lane % 4) + {0,1}; register 4j + {2,3}: the same columns 8 rows further down. =====
    float* C = p.C + (long long)split * p.c_split_stride;
    const int r0 = m0 + (wg - 1) * 64 + warp * 16 + (lane >> 2);
    const int cbase = n0 + 2 * (lane & 3);
    // every load of the epilogue is issued before the first store: one L2 round trip per tile, not one per column pair
    float2 bias[TC_BN / 8];
    int2 eb[TC_BN / 8];
    int ea[2] = {0, 0};
#pragma unroll
    for (int j = 0; j < TC_BN / 8; ++j) {
      bias[j] = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + cbase + 8 * j)) : make_float2(0.f, 0.f);
      eb[j] = F16 ? __ldg(reinterpret_cast<const int2*>(p.eb + cbase + 8 * j)) : make_int2(0, 0);
    }
    if constexpr (F16) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
        ea[h] = r0 + 8 * h < p.M ? (LDG_EA ? __ldg(p.ea + r0 + 8 * h) : __ldcg(p.ea + r0 + 8 * h)) : 0;
    }
#pragma unroll
    for (int j = 0; j < TC_BN / 8; ++j) {
      const int col = cbase + 8 * j;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        float x = acc[4 * j + 2 * h], y = acc[4 * j + 2 * h + 1];
        if constexpr (F16) {
          x = unscale(x, ea[h] + eb[j].x);
          y = unscale(y, ea[h] + eb[j].y);
        }
        if (row < p.M) *reinterpret_cast<float2*>(C + (long long)row * p.ldc + col) = make_float2(x + bias[j].x, y + bias[j].y);
      }
    }
  }
}

__device__ __forceinline__ void init_ring(unsigned long long* bars) {
  for (int s = 0; s < TC_STAGES; ++s) {
    bar_init(smem_addr(&bars[s]), 1);
    bar_init(smem_addr(&bars[TC_STAGES + s]), 2);
  }
}

// F16 = false: tf32 hi/lo operands (m64n128k8); F16 = true: fp16 head/tail operands of rows and columns scaled by 2^ea,
// 2^eb (m64n128k16), unscaled in the epilogue.
// Persistent: each CTA walks the output tiles blockIdx.x, + gridDim.x, ... (N tiles fastest, then M tiles, then
// splits), and the ring of stages runs on across tiles, so that the producer fills the next tile's first stages while
// the consumers store the last one.
template <bool F16>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
               const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo,
               TcGemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B needs 1024-byte aligned tiles
  uint8_t* tiles = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int BK = F16 ? TC_BK_F16 : TC_BK;           // values per 128-byte row
  unsigned long long* bars = reinterpret_cast<unsigned long long*>(tiles + (size_t)TC_STAGES * TC_STAGE_BYTES);
  // bars[0..S): full (TMA bytes landed), bars[S..2S): empty (both consumer warpgroups are done with the slot)

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int total_kb = p.K / BK;

  if (threadIdx.x == 0) {
    init_ring(bars);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  uint32_t it = 0;
  if (wg == 0) {
    // ===== TMA producer =====
    if (t == 0) {
      for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
        const int n0 = (tile % p.tiles_n) * TC_BN, m0 = (tile / p.tiles_n % p.tiles_m) * TC_BM;
        const int kb0 = tile / (p.tiles_n * p.tiles_m) * p.kb_per_split;
        load_tile<BK>(&map_a_hi, &map_a_lo, &map_b_hi, &map_b_lo, tiles, bars, m0, n0, kb0,
                      min(p.kb_per_split, total_kb - kb0), it);
      }
    }
    return;
  }
  for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) mma_store_tile<F16, true>(p, tiles, bars, tile, wg, t, it);
}

// ---- fp16 operands: power-of-two range scaling and the head/tail split -------------------------------------------------
// Exponent e that puts max_abs * 2^e into [2^13, 2^14): 140 - the biased exponent of max_abs.  All-zero vectors get 0;
// e <= 127 keeps 2^e a normal float (vectors whose largest value is below 2^-114 are scaled less far), and e >= -115
// holds for every finite max_abs, so x * 2^e is exact and the epilogue's unscale by 2^-(e_row + e_col) is too.
__device__ __forceinline__ int f16_range_exponent(float max_abs) {
  if (max_abs == 0.f) return 0;
  return min(140 - (int)((__float_as_uint(max_abs) >> 23) & 0xFFu), 127);
}
__device__ __forceinline__ float exp2_int(int e) { return __uint_as_float((uint32_t)(e + 127) << 23); }   // e in [-126, 127]
// y = x * 2^e = head + tail: |y| < 2^14 keeps head finite, y - head is exact in fp32
__device__ __forceinline__ void split_f16(float y, __half& head, __half& tail) {
  head = __float2half_rn(y);
  tail = __float2half_rn(y - __half2float(head));
}

// one warp per row of x [M, K] (K % 64 == 0): e[r], head / tail [M, K] of row r scaled by 2^e[r]
__global__ void split_rows_f16_kernel(const float* __restrict__ x, __half* __restrict__ head, __half* __restrict__ tail,
                                      int* __restrict__ e, long long M, int K) {
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= M) return;
  const float2* row = reinterpret_cast<const float2*>(x + r * K);
  float mx = 0.f;
  for (int i = lane; i < K / 2; i += 32) {
    const float2 v = row[i];
    mx = fmaxf(mx, fmaxf(fabsf(v.x), fabsf(v.y)));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  const int er = f16_range_exponent(mx);
  const float s = exp2_int(er);
  if (lane == 0) e[r] = er;
  __half2* h2 = reinterpret_cast<__half2*>(head + r * K);
  __half2* t2 = reinterpret_cast<__half2*>(tail + r * K);
  for (int i = lane; i < K / 2; i += 32) {             // the row is in L1 from the first pass
    const float2 v = row[i];
    __half hx, hy, tx, ty;
    split_f16(v.x * s, hx, tx);
    split_f16(v.y * s, hy, ty);
    h2[i] = __halves2half2(hx, hy);
    t2[i] = __halves2half2(tx, ty);
  }
}

// ---- streamed fp16 projection ---------------------------------------------------------------------------------------
// The fork GEMM of encoder layer l + 1 while the BiGRU scan of layer l still runs (api.cu: run_encoder).  Input frame t
// of layer l + 1 is final once the forward scan has stored step t and the backward scan step T - 1 - t (a forward-only
// scan: once it has stored step t); the scan publishes how many steps each of its CTAs has stored (bigru.cu).
// gemm_f16_stream_kernel is gemm_tc_kernel<true> with a dynamic tile schedule: warps 1..3 of the producer warpgroup
// claim output tiles from one counter, in the order their rows become final (two directions: the middle m-tile first,
// then outward; forward only: m-tile 0 first, then upward), split the tile's rows of A into fp16 head / tail planes and
// exponents (split_rows_f16_kernel's rule) and hand the tile to the TMA thread and the consumers through a one-slot
// queue; the split of an m-tile is shared out in 8-row chunks among the CTAs that claim its n-tiles.  Launched beside
// the scan it claims only tiles whose rows are final and stops claiming when the scan has finished or has not
// progressed for spin_limit polls; a second, stream-ordered launch on every SM (progress == null) runs the rest.
// Every tile is computed exactly as gemm_tc_kernel<true> computes it, so the result does not depend on which launch did
// which tile.
constexpr int STREAM_CHUNK = 8;                          // rows per split work item
constexpr int STREAM_CHUNKS = TC_BM / STREAM_CHUNK;      // ... per m-tile
constexpr int STREAM_MAX_K = 1024;                       // a lane holds K / 128 float4 of each of two rows
constexpr int STREAM_PROGRESS_MAX = 1024;                // scan CTAs that can publish progress

struct StreamSched {
  const float* A;          // [M, K] fp32 rows
  __half *a_head, *a_tail; // [M, K] split planes (p.ea: the row exponents)
  const int* progress;     // [nscan] steps stored per scan CTA; null: every row is final
  int nscan, scan_cs;      // scan CTA i runs direction (i / scan_cs) % ndir
  int ndir;                // 1: every scan CTA runs forward (no backward progress to wait for)
  int T, k, B;             // frames scanned, subsampling (output frame f = scan frame f k), batch rows per frame
  int mid;                 // m-tile whose rows become final first
  unsigned spin_limit;     // polls without progress before a launch beside the scan stops claiming
  int* claim;              // next claim index
  int* chunk_next;         // [tiles_m] split chunks handed out
  int* chunk_done;         // [tiles_m] split chunks finished
  int* tiles_done;         // tiles this launch claimed are added here
  int* claims;             // [3 tiles] or null: (m-tile + 1, fwd, bwd) of each tile claimed beside the scan, with the
                           // progress its rows were found final at
};

__device__ __forceinline__ int ld_acquire_i32(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.b32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ int ld_relaxed_i32(const int* p) {
  int v;
  asm volatile("ld.relaxed.gpu.global.b32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// generic-proxy writes of the split planes <-> TMA (async-proxy) reads of them
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;\n" ::: "memory"); }
__device__ __forceinline__ void named_sync(int id, int count) { asm volatile("bar.sync %0, %1;\n" ::"r"(id), "r"(count) : "memory"); }
// mbarrier wait without the trap of bar_wait: the tile queue may wait for as long as the scan takes to make rows final
__device__ __forceinline__ void bar_wait_sleep(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    if (ok) break;
    __nanosleep(64);
  }
}

// claim index i (in units of whole m-tiles) -> m-tile: mid, then alternately one further right and one further left
__device__ __forceinline__ int stream_m_tile(int i, int mid, int tiles_m) {
  if (i == 0) return mid;
  const int j = i - 1, left = mid, right = tiles_m - 1 - mid, both = min(left, right);
  if (j < 2 * both) return (j & 1) ? mid - 1 - (j >> 1) : mid + 1 + (j >> 1);
  return right > left ? mid + 1 + j - both : mid - 1 - (j - both);
}

// One warp: the fewest steps any forward / backward scan CTA has published; spins counts the polls since they changed
__device__ __forceinline__ void stream_poll(const StreamSched& s, int lane, int& fwd, int& bwd, unsigned& spins) {
  int f = INT_MAX, b = INT_MAX;
  for (int i = lane; i < s.nscan; i += 32) {
    const int v = ld_acquire_i32(s.progress + i);
    if (s.ndir == 2 && ((i / s.scan_cs) & 1)) b = min(b, v); else f = min(f, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    f = min(f, __shfl_xor_sync(0xffffffffu, f, o));
    b = min(b, __shfl_xor_sync(0xffffffffu, b, o));
  }
  spins = (f == fwd && b == bwd) ? spins + 1 : 0;
  fwd = f;
  bwd = b;
}
__device__ __forceinline__ bool stream_ready(const StreamSched& s, const TcGemmParams& p, int c, int fwd, int bwd) {
  const int m = stream_m_tile(c / p.tiles_n, s.mid, p.tiles_m);
  const int r0 = m * TC_BM, r1 = min(r0 + TC_BM, p.M) - 1;
  return fwd >= (r1 / s.B) * s.k + 1 && bwd >= s.T - (r0 / s.B) * s.k;
}

// One warp: claims the next tile (-1: none for this launch).  Beside the scan (s.progress set) a tile is claimed only
// once the next one in claim order has its rows final, and no tile once the scan has finished or has not progressed for
// spin_limit polls.  fwd / bwd / spins: stream_poll's state; polls_due: claims so far.
__device__ int stream_claim(const StreamSched& s, const TcGemmParams& p, int lane, int& fwd, int& bwd, unsigned& spins,
                           unsigned& polls_due) {
  const int total = p.tiles_m * p.tiles_n;
  if (!s.progress) {
    const int c = __shfl_sync(0xffffffffu, lane == 0 ? atomicAdd(s.claim, 1) : 0, 0);
    return c < total ? c : -1;
  }
  // the progress words are polled only when the last answer does not cover the next tile, and at every 4th claim to
  // notice the end of the scan: every poll is 2 loads per lane of lines the scan writes
  bool poll = (++polls_due & 3) == 0;
  while (true) {
    if (poll) stream_poll(s, lane, fwd, bwd, spins);
    // the scan is done (or stalled and was waited for below): the launch on every SM takes the rest
    if (fwd >= s.T && bwd >= s.T) return -1;
    const int head = __shfl_sync(0xffffffffu, lane == 0 ? ld_relaxed_i32(s.claim) : 0, 0);
    if (head >= total) return -1;
    if (stream_ready(s, p, head, fwd, bwd)) break;
    if (poll && spins >= s.spin_limit) return -1;
    if (poll) __nanosleep(256);
    poll = true;
  }
  const int c = __shfl_sync(0xffffffffu, lane == 0 ? atomicAdd(s.claim, 1) : 0, 0);
  if (c >= total) return -1;
  // other CTAs may have claimed the tiles up to c since the head was seen final: c follows within a few steps
  while (!stream_ready(s, p, c, fwd, bwd)) {
    if (spins >= s.spin_limit) {
      // the scan stalls: this tile is claimed, so wait for the scan to end (its rows are final then); fwd = bwd = T
      // makes the next stream_claim of this warp return -1, so the CTA stops after this tile
      asm volatile("griddepcontrol.wait;\n" ::: "memory");
      fwd = bwd = s.T;
      break;
    }
    __nanosleep(256);
    stream_poll(s, lane, fwd, bwd, spins);
  }
  if (lane == 0 && s.claims) {
    s.claims[3LL * c] = stream_m_tile(c / p.tiles_n, s.mid, p.tiles_m) + 1;
    s.claims[3LL * c + 1] = fwd;
    s.claims[3LL * c + 2] = bwd;
  }
  return c;
}

// rows r0, r0 + 1 of A (r < M): exponent, head, tail -- split_rows_f16_kernel's rule, with both rows' loads in flight
// at once and every load from L2 (other SMs wrote A while this kernel runs)
__device__ __forceinline__ void stream_split_pair(const StreamSched& s, int* ea, long long r0, long long M, int K, int lane) {
  constexpr int MAXV = STREAM_MAX_K / 128;
  const int nv = K / 128;
  float4 v[2][MAXV];
#pragma unroll
  for (int q = 0; q < 2; ++q)
#pragma unroll
    for (int i = 0; i < MAXV; ++i)
      if (i < nv && r0 + q < M) v[q][i] = __ldcg(reinterpret_cast<const float4*>(s.A + (r0 + q) * K) + lane + 32 * i);
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    if (r0 + q >= M) break;
    float mx = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i)
      if (i < nv) mx = fmaxf(mx, fmaxf(fmaxf(fabsf(v[q][i].x), fabsf(v[q][i].y)), fmaxf(fabsf(v[q][i].z), fabsf(v[q][i].w))));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const int er = f16_range_exponent(mx);
    const float sc = exp2_int(er);
    if (lane == 0) ea[r0 + q] = er;
    uint2* h = reinterpret_cast<uint2*>(s.a_head + (r0 + q) * K);
    uint2* tl = reinterpret_cast<uint2*>(s.a_tail + (r0 + q) * K);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      if (i >= nv) break;
      __half hx, hy, hz, hw, tx, ty, tz, tw;
      split_f16(v[q][i].x * sc, hx, tx);
      split_f16(v[q][i].y * sc, hy, ty);
      split_f16(v[q][i].z * sc, hz, tz);
      split_f16(v[q][i].w * sc, hw, tw);
      const __half2 h01 = __halves2half2(hx, hy), h23 = __halves2half2(hz, hw);
      const __half2 t01 = __halves2half2(tx, ty), t23 = __halves2half2(tz, tw);
      h[lane + 32 * i] = make_uint2(*reinterpret_cast<const uint32_t*>(&h01), *reinterpret_cast<const uint32_t*>(&h23));
      tl[lane + 32 * i] = make_uint2(*reinterpret_cast<const uint32_t*>(&t01), *reinterpret_cast<const uint32_t*>(&t23));
    }
  }
}

// One warp: takes 8-row chunks of m-tile m until none is left, then waits until every chunk (its own and those other
// warps or CTAs took) is split
__device__ __forceinline__ void stream_split_tile(const StreamSched& s, const TcGemmParams& p, int m, int lane) {
  while (true) {
    const int ch = __shfl_sync(0xffffffffu, lane == 0 ? atomicAdd(s.chunk_next + m, 1) : 0, 0);
    if (ch >= STREAM_CHUNKS) break;
    const long long r = (long long)m * TC_BM + ch * STREAM_CHUNK;
    for (int q = 0; q < STREAM_CHUNK; q += 2) stream_split_pair(s, const_cast<int*>(p.ea), r + q, p.M, p.K, lane);
    fence_proxy_async_global();
    __syncwarp();
    if (lane == 0) {
      __threadfence();
      atomicAdd(s.chunk_done + m, 1);
    }
  }
  if (lane == 0)
    while (ld_acquire_i32(s.chunk_done + m) < STREAM_CHUNKS) __nanosleep(128);
  __syncwarp();
}

__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_f16_stream_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                       const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo,
                       TcGemmParams p, StreamSched s) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* tiles = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  unsigned long long* bars = reinterpret_cast<unsigned long long*>(tiles + (size_t)TC_STAGES * TC_STAGE_BYTES);
  // bars[0..2S): the ring as in gemm_tc_kernel; bars[2S]: a tile id is in the queue slot, bars[2S + 1]: the TMA thread
  // and all 256 consumer threads have read it
  volatile int* q_tile = reinterpret_cast<volatile int*>(bars + 2 * TC_STAGES + 2);
  volatile int* q_claim = q_tile + 1;
  const uint32_t q_full = smem_addr(&bars[2 * TC_STAGES]), q_empty = smem_addr(&bars[2 * TC_STAGES + 1]);
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    init_ring(bars);
    bar_init(q_full, 1);
    bar_init(q_empty, 1 + 256);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  uint32_t it = 0;
  if (warp == 0) {
    // ===== TMA thread =====
    if (lane == 0) {
      for (uint32_t n = 0;; ++n) {
        bar_wait_sleep(q_full, n & 1u);
        const int tile = *q_tile;
        bar_arrive(q_empty);
        if (tile < 0) break;
        fence_proxy_async_global();
        load_tile<TC_BK_F16>(&map_a_hi, &map_a_lo, &map_b_hi, &map_b_lo, tiles, bars, (tile / p.tiles_n) * TC_BM,
                             (tile % p.tiles_n) * TC_BN, 0, p.K / TC_BK_F16, it);
      }
    }
  } else if (wg == 0) {
    // ===== warps 1..3: claim, split, queue =====
    int fwd = -1, bwd = -1, claimed = 0;
    unsigned spins = 0, polls_due = 0;
    for (uint32_t n = 0;; ++n) {
      bar_wait_sleep(q_empty, (n & 1u) ^ 1u);            // the slot is free (first round passes immediately)
      if (warp == 1) {
        const int c = stream_claim(s, p, lane, fwd, bwd, spins, polls_due);
        if (lane == 0) *q_claim = c;
      }
      named_sync(1, 96);
      const int c = *q_claim;
      int tile = -1;
      if (c >= 0) {
        const int m = stream_m_tile(c / p.tiles_n, s.mid, p.tiles_m);
        tile = m * p.tiles_n + c % p.tiles_n;
        stream_split_tile(s, p, m, lane);
      }
      named_sync(1, 96);                                   // q_claim read by all, every chunk of the tile split
      if (warp == 1 && lane == 0) {
        *q_tile = tile;
        bar_arrive(q_full);
      }
      if (c < 0) break;
      ++claimed;
    }
    if (warp == 1 && lane == 0 && claimed) atomicAdd(s.tiles_done, claimed);
  } else {
    // ===== consumers =====
    for (uint32_t n = 0;; ++n) {
      bar_wait_sleep(q_full, n & 1u);
      const int tile = *q_tile;
      bar_arrive(q_empty);
      if (tile < 0) break;
      mma_store_tile<true, false>(p, tiles, bars, tile, wg, t, it);
    }
  }
  // launched beside the scan: this kernel completes only after the scan has (no-op for a stream-ordered launch).  The
  // whole warp waits together: lanes that reached the wait early would otherwise hold back a lane still issuing loads.
  __syncwarp();
  asm volatile("griddepcontrol.wait;\n" ::: "memory");
}

// W [K, N] row-major -> K-major head / tail [N, K] of every column n scaled by 2^e[n] (weights, once per finalize).
// One block of 32 x 8 threads per 32 columns: the column maxima first, then 32 x 32 tiles through shared memory.
__global__ void transpose_split_f16_kernel(const float* __restrict__ W, __half* __restrict__ head, __half* __restrict__ tail,
                                           int* __restrict__ e, int K, int N) {
  __shared__ float tile[32][33];
  __shared__ float scale[32];
  const int n0 = blockIdx.x * 32, tx = threadIdx.x, ty = threadIdx.y;
  const int n = n0 + tx;
  float mx = 0.f;
  if (n < N)
    for (int k = ty; k < K; k += 8) mx = fmaxf(mx, fabsf(W[(long long)k * N + n]));
  tile[ty][tx] = mx;
  __syncthreads();
  if (ty == 0) {
    for (int i = 1; i < 8; ++i) mx = fmaxf(mx, tile[i][tx]);
    const int en = f16_range_exponent(mx);
    if (n < N) e[n] = en;
    scale[tx] = exp2_int(en);
  }
  __syncthreads();
  for (int k0 = 0; k0 < K; k0 += 32) {
    for (int i = ty; i < 32; i += 8) {
      const int k = k0 + i;
      tile[i][tx] = (k < K && n < N) ? W[(long long)k * N + n] * scale[tx] : 0.f;
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
      const int nn = n0 + i, k = k0 + tx;
      if (nn < N && k < K) split_f16(tile[tx][i], head[(long long)nn * K + k], tail[(long long)nn * K + k]);
    }
    __syncthreads();
  }
}

// x = hi + lo with both parts exactly representable in tf32
__global__ void split_tf32_kernel(const float4* __restrict__ x, float4* __restrict__ hi, float4* __restrict__ lo,
                                  long long n4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = x[i];
    float4 h, l;
    auto split = [](float a, float& ah, float& al) {
      ah = __uint_as_float(__float_as_uint(a) & 0xFFFFE000u);
      const float r = a - ah;
      uint32_t t;
      asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(t) : "f"(r));
      al = __uint_as_float(t);
    };
    split(v.x, h.x, l.x); split(v.y, h.y, l.y); split(v.z, h.z, l.z); split(v.w, h.w, l.w);
    hi[i] = h;
    lo[i] = l;
  }
}

// [K, N] row-major -> K-major [N, K] hi/lo pair (weights, once per finalize)
__global__ void transpose_split_kernel(const float* __restrict__ W, float* __restrict__ hi, float* __restrict__ lo,
                                       int K, int N, int Kpad, int ldw) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = k0 + i, n = n0 + threadIdx.x;
    tile[i][threadIdx.x] = (k < K && n < N) ? W[(long long)k * ldw + n] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int n = n0 + i, k = k0 + threadIdx.x;
    if (n < N && k < Kpad) {                      // k in [K, Kpad): zero padding of the contraction dimension
      const float a = tile[threadIdx.x][i];
      const float ah = __uint_as_float(__float_as_uint(a) & 0xFFFFE000u);
      uint32_t t;
      asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(t) : "f"(a - ah));
      hi[(long long)n * Kpad + k] = ah;
      lo[(long long)n * Kpad + k] = __uint_as_float(t);
    }
  }
}

// split + zero-pad the contraction dimension in one pass: x [M, K] -> hi / lo [M, Kpad] (layer 0: K = 40 -> 64)
__global__ void split_pad_tf32_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo,
                                      long long M, int K, int Kpad) {
  const long long total = M * Kpad;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / Kpad;
    const int k = (int)(i % Kpad);
    const float a = k < K ? x[r * K + k] : 0.f;
    const float ah = __uint_as_float(__float_as_uint(a) & 0xFFFFE000u);
    uint32_t t;
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(t) : "f"(a - ah));
    hi[i] = ah;
    lo[i] = __uint_as_float(t);
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

int get_encode() {
  if (g_encode) return 0;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  LVSR_CUDA_OK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  LVSR_CHECK(fn != nullptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available");
  g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  return 0;
}

// 2-D fp32 or fp16 tensor [rows, K] (K contiguous), box = [128 rows, one 128-byte row: 32 floats or 64 halves],
// 128-byte swizzle
int make_map(CUtensorMap* map, const void* ptr, long long rows, int K, bool f16) {
  const size_t esize = f16 ? sizeof(__half) : sizeof(float);
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)K * esize};
  cuuint32_t box[2] = {(cuuint32_t)(128 / esize), (cuuint32_t)TC_BM};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(map, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                        const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  LVSR_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return 0;
}

// C = A . B^T (+ bias) on the presplit K-major operands of either kind; K is a multiple of the kind's k-block
template <bool F16>
int launch_tc(const void* A_hi, const void* A_lo, const int* ea, int M, const void* B_hi, const void* B_lo, const int* eb,
              int N, int K, const float* bias, float* C, int ldc, int splits, long long split_stride, cudaStream_t stream) {
  ProfScope prof("gemm", stream);
  constexpr int BK = F16 ? TC_BK_F16 : TC_BK;
  LVSR_CHECK(M >= 1 && N % TC_BN == 0 && K % BK == 0 && K >= BK && splits >= 1,
             "gemm_tc: unsupported shape M=%d N=%d K=%d (%s operands)", M, N, K, F16 ? "fp16" : "tf32");
  if (int rc = get_encode()) return rc;
  CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
  if (int rc = make_map(&ma_hi, A_hi, M, K, F16)) return rc;
  if (int rc = make_map(&ma_lo, A_lo, M, K, F16)) return rc;
  if (int rc = make_map(&mb_hi, B_hi, N, K, F16)) return rc;
  if (int rc = make_map(&mb_lo, B_lo, N, K, F16)) return rc;
  static bool configured[LVSR_MAX_DEVICES] = {false};
  const int dev = current_device();
  if (!configured[dev]) {
    LVSR_CUDA_OK(cudaFuncSetAttribute(gemm_tc_kernel<F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_SMEM));
    configured[dev] = true;
  }
  const int total_kb = K / BK;
  splits = std::min(splits, total_kb);
  TcGemmParams p;
  p.C = C; p.bias = bias; p.ea = ea; p.eb = eb; p.M = M; p.N = N; p.K = K; p.ldc = ldc;
  p.kb_per_split = ceil_div(total_kb, splits);
  p.c_split_stride = split_stride;
  p.tiles_n = N / TC_BN;
  p.tiles_m = ceil_div(M, TC_BM);
  const long long tiles = (long long)p.tiles_n * p.tiles_m * ceil_div(total_kb, p.kb_per_split);
  LVSR_CHECK(tiles <= INT32_MAX, "gemm_tc: too many tiles (M=%d N=%d)", M, N);
  p.tiles = (int)tiles;
  // one CTA per SM (TC_SMEM), each walking tiles
  const int grid = (int)std::min<long long>(tiles, device_sm_count());
  gemm_tc_kernel<F16><<<grid, TC_THREADS, TC_SMEM, stream>>>(ma_hi, ma_lo, mb_hi, mb_lo, p);
  LVSR_LAUNCH_CHECK();
  return 0;
}

}  // namespace

// the contraction dimension is zero-padded to a multiple of the 32-float TMA box (layer 0: K = 40 -> 64)
int gemm_tc_kpad(int K) { return ceil_div(K, TC_BK) * TC_BK; }

bool gemm_tc_supported(int M, int N, int K) {
  return M >= 1 && N % TC_BN == 0 && K >= 4 && K % 4 == 0;
}

// Wt_hi / Wt_lo: [N, gemm_tc_kpad(K)]
int split_weight_tf32(const float* W, int K, int N, float* Wt_hi, float* Wt_lo, cudaStream_t stream) {
  const int Kpad = gemm_tc_kpad(K);
  dim3 grid(ceil_div(N, 32), ceil_div(Kpad, 32)), block(32, 8);
  transpose_split_kernel<<<grid, block, 0, stream>>>(W, Wt_hi, Wt_lo, K, N, Kpad, N);
  LVSR_LAUNCH_CHECK();
  return 0;
}

// [K rows, N columns, leading dimension ldw] -> K-major hi/lo [N, gemm_tc_kpad(K)] (operands of the TN product)
int transpose_split_tf32(const float* W, int K, int N, int ldw, float* hi, float* lo, cudaStream_t stream) {
  const int Kpad = gemm_tc_kpad(K);
  dim3 grid(ceil_div(N, 32), ceil_div(Kpad, 32)), block(32, 8);
  LVSR_CHECK(grid.y <= 65535, "transpose_split: too many rows (%d)", K);
  transpose_split_kernel<<<grid, block, 0, stream>>>(W, hi, lo, K, N, Kpad, ldw);
  LVSR_LAUNCH_CHECK();
  return 0;
}

// element-wise exact split x = hi + lo (n % 4 == 0)
int split_tf32(const float* x, float* hi, float* lo, long long n, cudaStream_t stream) {
  const long long n4 = n / 4;
  split_tf32_kernel<<<(int)std::min<long long>(4096, (n4 + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(hi), reinterpret_cast<float4*>(lo), n4);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int gemm_tc_splits_launched(int Kpad, int splits) {
  const int total_kb = Kpad / TC_BK;
  splits = std::max(1, std::min(splits, total_kb));
  return ceil_div(total_kb, ceil_div(total_kb, splits));
}

// C[M,N] (+ bias) = A . B^T with both operands K-major hi/lo pairs: A [M, Kpad], B [N, Kpad].  splits > 1: split-K, partial
// result z goes to C + z * split_stride (the caller adds them up).
int gemm_tc_presplit(const float* A_hi, const float* A_lo, int M, const float* B_hi, const float* B_lo, int N, int Kpad,
                     const float* bias, float* C, int ldc, int splits, long long split_stride, cudaStream_t stream) {
  return launch_tc<false>(A_hi, A_lo, nullptr, M, B_hi, B_lo, nullptr, N, Kpad, bias, C, ldc, splits, split_stride, stream);
}

// C[M,N] = A[M,K] . W + bias with W given as the K-major hi/lo pair produced by split_weight_tf32.
// A_hi / A_lo: caller-provided scratch of M * gemm_tc_kpad(K) floats each.
int gemm_tc(const float* A, float* A_hi, float* A_lo, int M, int K, const float* Wt_hi, const float* Wt_lo, int N,
            const float* bias, float* C, int ldc, cudaStream_t stream) {
  LVSR_CHECK(gemm_tc_supported(M, N, K), "gemm_tc: unsupported shape M=%d N=%d K=%d", M, N, K);
  if (int rc = get_encode()) return rc;
  const int Kpad = gemm_tc_kpad(K);
  if (Kpad == K) {
    const long long n4 = (long long)M * K / 4;
    split_tf32_kernel<<<(int)std::min<long long>(4096, (n4 + 255) / 256), 256, 0, stream>>>(
        reinterpret_cast<const float4*>(A), reinterpret_cast<float4*>(A_hi), reinterpret_cast<float4*>(A_lo), n4);
  } else {
    const long long n = (long long)M * Kpad;
    split_pad_tf32_kernel<<<(int)std::min<long long>(4096, (n + 255) / 256), 256, 0, stream>>>(A, A_hi, A_lo, M, K, Kpad);
  }
  LVSR_LAUNCH_CHECK();
  return gemm_tc_presplit(A_hi, A_lo, M, Wt_hi, Wt_lo, N, Kpad, bias, C, ldc, 1, 0, stream);
}

bool gemm_f16_supported(int M, int N, int K) { return M >= 1 && N % TC_BN == 0 && K >= TC_BK_F16 && K % TC_BK_F16 == 0; }

// W [K, N] row-major -> Wt_head / Wt_tail [N, K] halves and ew [N]
int split_weight_f16(const float* W, int K, int N, __half* Wt_head, __half* Wt_tail, int* ew, cudaStream_t stream) {
  LVSR_CHECK(K % TC_BK_F16 == 0 && K > 0 && N > 0, "split_weight_f16: unsupported shape K=%d N=%d", K, N);
  transpose_split_f16_kernel<<<ceil_div(N, 32), dim3(32, 8), 0, stream>>>(W, Wt_head, Wt_tail, ew, K, N);
  LVSR_LAUNCH_CHECK();
  return 0;
}

// C[M,N] = A[M,K] . W + bias on fp16 head/tail operands, W as split_weight_f16 left it.  A_head / A_tail (M * K halves
// each) and ea (M ints): caller-provided scratch for the split of A.
int gemm_f16(const float* A, __half* A_head, __half* A_tail, int* ea, int M, int K, const __half* Wt_head,
             const __half* Wt_tail, const int* ew, int N, const float* bias, float* C, int ldc, cudaStream_t stream) {
  LVSR_CHECK(gemm_f16_supported(M, N, K), "gemm_f16: unsupported shape M=%d N=%d K=%d", M, N, K);
  constexpr int ROWS_PER_BLOCK = 8;
  split_rows_f16_kernel<<<ceil_div(M, ROWS_PER_BLOCK), 32 * ROWS_PER_BLOCK, 0, stream>>>(
      A, A_head, A_tail, ea, M, K);
  LVSR_LAUNCH_CHECK();
  return launch_tc<true>(A_head, A_tail, ea, M, Wt_head, Wt_tail, ew, N, K, bias, C, ldc, 1, 0, stream);
}

// stream_split_pair moves whole float4 groups, K / 128 per lane and row
bool gemm_f16_stream_supported(int M, int N, int K) {
  return gemm_f16_supported(M, N, K) && K % 128 == 0 && K <= STREAM_MAX_K;
}

// [claim | pad | progress [STREAM_PROGRESS_MAX] | chunk_next [tiles_m] | chunk_done [tiles_m]]
size_t gemm_f16_stream_sync_ints(int M) { return 32 + STREAM_PROGRESS_MAX + 2 * (size_t)ceil_div(M, TC_BM); }
int* gemm_f16_stream_progress(int* sync) { return sync + 32; }
int gemm_f16_stream_max_scan_ctas() { return STREAM_PROGRESS_MAX; }

int gemm_f16_stream(const float* A, __half* A_head, __half* A_tail, int* ea, int M, int K, const __half* Wt_head,
                    const __half* Wt_tail, const int* ew, int N, const float* bias, float* C, int ldc,
                    const ProjStream& ps, int grid, cudaStream_t stream) {
  LVSR_CHECK(gemm_f16_stream_supported(M, N, K) && ps.nscan <= STREAM_PROGRESS_MAX && grid >= 1 && ps.k >= 1 &&
                 (long long)ceil_div(ps.T, ps.k) * ps.B == M,
             "gemm_f16_stream: unsupported shape M=%d N=%d K=%d (T=%d k=%d B=%d)", M, N, K, ps.T, ps.k, ps.B);
  if (int rc = get_encode()) return rc;
  CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
  if (int rc = make_map(&ma_hi, A_head, M, K, true)) return rc;
  if (int rc = make_map(&ma_lo, A_tail, M, K, true)) return rc;
  if (int rc = make_map(&mb_hi, Wt_head, N, K, true)) return rc;
  if (int rc = make_map(&mb_lo, Wt_tail, N, K, true)) return rc;
  static bool configured[LVSR_MAX_DEVICES] = {false};
  const int dev = current_device();
  if (!configured[dev]) {
    LVSR_CUDA_OK(cudaFuncSetAttribute(gemm_f16_stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_SMEM));
    configured[dev] = true;
  }
  TcGemmParams p;
  p.C = C; p.bias = bias; p.ea = ea; p.eb = ew; p.M = M; p.N = N; p.K = K; p.ldc = ldc;
  p.kb_per_split = K / TC_BK_F16;
  p.c_split_stride = 0;
  p.tiles_n = N / TC_BN;
  p.tiles_m = ceil_div(M, TC_BM);
  LVSR_CHECK((long long)p.tiles_n * p.tiles_m <= INT32_MAX, "gemm_f16_stream: too many tiles (M=%d N=%d)", M, N);
  p.tiles = p.tiles_n * p.tiles_m;
  StreamSched s;
  s.A = A; s.a_head = A_head; s.a_tail = A_tail;
  s.progress = ps.progress;
  s.nscan = ps.nscan; s.scan_cs = ps.scan_cs; s.ndir = ps.ndir; s.T = ps.T; s.k = ps.k; s.B = ps.B;
  // the frame that becomes final first: the fewest scan steps max(f k + 1, T - f k) that both directions need, or
  // f k + 1 when the scan runs forward only (frame 0, so the m-tiles are claimed in ascending order)
  int best = INT_MAX, fmid = 0;
  for (int f = 0; f * ps.k < ps.T; ++f) {
    const int ready = ps.ndir == 1 ? f * ps.k + 1 : std::max(f * ps.k + 1, ps.T - f * ps.k);
    if (ready < best) { best = ready; fmid = f; }
  }
  s.mid = std::min((int)((long long)fmid * ps.B / TC_BM), p.tiles_m - 1);
  s.spin_limit = ps.spin_limit;
  s.claim = ps.sync;
  s.chunk_next = ps.sync + 32 + STREAM_PROGRESS_MAX;
  s.chunk_done = s.chunk_next + p.tiles_m;
  s.tiles_done = ps.tiles_done;
  s.claims = ps.progress ? ps.claims : nullptr;
  // beside the scan: a programmatic dependent launch, started once every scan CTA runs (griddepcontrol.launch_dependents
  // after its entry barrier), so its CTAs only take SMs the scan does not need
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(std::min(grid, p.tiles));
  cfg.blockDim = dim3(TC_THREADS);
  cfg.dynamicSmemBytes = TC_SMEM;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = ps.progress ? 1 : 0;
  LVSR_CUDA_OK(cudaLaunchKernelEx(&cfg, gemm_f16_stream_kernel, ma_hi, ma_lo, mb_hi, mb_lo, p, s));
  LVSR_LAUNCH_CHECK();
  return 0;
}

}  // namespace lvsr
