// Bidirectional GatedRecurrent scan of one encoder layer -- one persistent,
// cluster-resident kernel for BOTH directions of the layer.
//
// Replaces theano.scan over GatedRecurrent.apply for the forward and the backward
// child of Bidirectional (B/bricks/recurrent.py:224-231, 608-620, 655-663) plus the
// x[::k] subsampling of Encoder.apply (lvsr/bricks/__init__.py:75-77).
//
// Mapping (two DEPENDENT [rows,D]x[D,*] products per step, T sequential steps):
//   * batch rows are independent -> a thread-block CLUSTER of CS CTAs owns RB = 4 rows of one
//     direction; clusters never talk to each other (no grid-wide barrier).  The tensor-core kernel also comes with
//     RB = 8 rows per cluster, chosen when it needs fewer waves of clusters than RB = 4 (a cluster's CTAs must share one
//     GPC, so an H100 holds fewer 4-CTA clusters than SMs / 4; see bigru_layer).
//   * inside a cluster the hidden units are split: CTA `rank` owns UC = D/CS units, each of its
//     warps 4 of them; the state_to_gates slice stays IN REGISTERS for the whole sequence, the
//     state_to_state slice in shared memory -- weights are read from HBM once per layer.
//   * per step: gates for the owned units (needs all of h), all-gather of h*r, candidate for the
//     owned units, all-gather of h'.  An all-gather is one `st.async` per lane: 16 bytes go from
//     registers straight into the receiver's shared memory and credit the RECEIVER's mbarrier
//     (complete_tx); no staging buffer, no proxy fence, no CTA or cluster barrier in the loop --
//     a warp only ever waits for "all RB*D*4 bytes of h (or h*r) have landed".  h never leaves the chip.
//   * inside a warp k is split over 16 lanes and the warp's columns over the other 2 (see the kernel);
//     everything the epilogues need from other lanes travels by shuffle.
//   * the fork pre-activations of step t+1 are prefetched into registers during step t.
//   * TAPE (training): the gates / candidate overwrite the pre-activations they were computed from and every
//     frame of h is kept (hext), for the reverse-time scan of bigru_bwd.cu; compiled out of the inference kernel.
// The FFMA products are bound by the shared-memory return path of the h loads, the rest is lock-step latency.  Hidden
// size 256 runs bigru_mma_kernel below (mma.sync on fp16 head/tail splits, weights as the M dimension, warp-specialised);
// the FFMA kernel stays for the other hidden sizes and as the reference the tensor-core kernel is tested against.
#include <cuda_fp16.h>

#include "kernels.h"
#include "lvsr_b200.h"

namespace lvsr {

namespace {

constexpr int RB = 4;        // batch rows per cluster

// LVSR_BIGRU_TRACE=1: thread 0 of CTA 0 accumulates the SM clock spent in each section of a step
// (wait h, gate product, gate epilogue + send, wait h*r, candidate product, epilogue + send).
__device__ unsigned long long g_bigru_trace[12];
__device__ int g_bigru_trace_on = 0;
// per CTA: cycles from kernel entry to the first step, cycles inside the time loop (tensor-core kernel, trace runs only)
__device__ unsigned long long g_bigru_cta_cycles[2][1024];

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t map_to_rank(uint32_t local_addr, int rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;\n" : "=r"(remote) : "r"(local_addr), "r"(rank));
  return remote;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arm(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
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
    if (++spins > (1ull << 24)) __trap();   // a lost transfer must fail the launch, not hang the GPU
  }
}
// 16 bytes straight from registers into the shared memory of another CTA of the cluster; the
// RECEIVER's mbarrier is credited with the bytes when they land (no staging buffer, no proxy
// fence, no CTA barrier on the sender).
__device__ __forceinline__ void st_async_v4(uint32_t remote_addr, float x, float y, float z, float w,
                                            uint32_t remote_bar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1, %2, %3, %4}, [%5];\n" ::"r"(
                   remote_addr),
               "f"(x), "f"(y), "f"(z), "f"(w), "r"(remote_bar)
               : "memory");
}

// float4 groups of a lane's gate-weight k range (D / 64 of them) that the FFMA kernel keeps in registers: all of them at
// D = 64, 128 and 256 (as the kernel always did), one at the other widths -- two already spill at
// __launch_bounds__(256, 2), and the rolled loop over the shared-memory groups keeps their loads from being hoisted.
template <int D>
__host__ __device__ constexpr int ffma_qreg() { return D <= 128 || D == 256 ? D / 64 : 1; }

// D: hidden units per direction; CS: CTAs per cluster.
//
// Work split inside a warp: lane = kg * CG + cg.
//   kg (KL = 16 groups) owns the k range [kg * D/16, +D/16) of both products;
//   cg (CG = 2 groups)  owns half of the warp's gate columns (cg 0: the 4 update gates, cg 1: the 4
//                       reset gates) and half of its candidate columns.
// A lane accumulates RB x 4 gate sums and RB x 2 candidate sums over its D/16 k values; the
// cross-lane reduction runs over the 16 kg-lanes: 15 + 8 exchanges per step.  The split is a
// trade: every lane must read its k range of h for all rows, and the shared-memory RETURN path
// (128 B/clk/SM, 4 cycles per warp-wide 16-byte load) is what bounds a phase -- k over 8 lanes:
// 72 loads per warp and step; k over 32 lanes: 24 loads but 46 exchanges and ~1000 instructions
// per warp and step (issue-bound); 16 lanes sits between.
//
// Shapes: <D, D / 32 CTAs, 8 warps> = 256 threads for every D = 64, 128, ..., 512 (32 units per CTA, so 2 to 16 CTAs per
// cluster; above 8 the cluster size is non-portable), two CTAs (two different clusters) per SM where shared memory
// allows it (up to D = 192; the shared-memory weights of wider layers leave room for one CTA per SM).  At D = 64, 128
// and 256 a lane's gate slice (4 * D/16 floats) stays in registers; at the other widths the first float4 group of its
// k range does and the rest sits in shared memory beside the state_to_state slice (see ffma_qreg).
// NDIR: directions of the layer.  2: cluster c runs direction c & 1 on rows (c >> 1) * RB; 1 (net.bidir False): every
// cluster runs the forward direction, on rows c * RB, and the pre-activations, outputs and hext hold one direction.
// TAPE: training forward (stores c / z / r over the pre-activations and every frame of h); compiled out for inference
template <int D, int CS, int NDIR, int NWARP, bool TAPE>
__global__ void __launch_bounds__(NWARP * 32, 2)
bigru_kernel(BiGruArgs a) {
  constexpr int UC = D / CS;          // units owned by this CTA
  constexpr int KL = 16;              // lanes that split k
  constexpr int CG = 32 / KL;         // lanes that split the warp's columns
  constexpr int KPG = D / KL;         // k values per lane
  constexpr int KQ = KPG / 4;         // float4 groups per lane
  constexpr int NC2 = UC / NWARP;     // units per warp (candidate columns)
  constexpr int NC1 = 2 * NC2;        // gate columns per warp: [z units | r units]
  constexpr int CPL1 = NC1 / CG;      // gate columns per lane
  constexpr int CPL2 = NC2 / CG;      // candidate columns per lane
  static_assert(D % (CS * NWARP) == 0 && D % (4 * KL) == 0, "unsupported D / cluster size");
  static_assert(NC2 % CG == 0 && CPL2 == 2 && CPL1 == 4, "lane roles below assume 4 gate / 2 candidate columns per lane");
  static_assert(KPG <= 32, "a lane's k range sits inside one chunk of h");
  static_assert(CS <= 16, "sender lanes reach at most 16 peers");
  static_assert(NDIR == 1 || NDIR == 2, "one or two directions");
  constexpr int QREG = ffma_qreg<D>();   // float4 groups of the gate slice held in registers, the rest in shared memory
  constexpr int N1 = RB * CPL1, N2 = RB * CPL2;        // per-lane partial sums of the two phases
  constexpr uint32_t FULL_BYTES = RB * D * sizeof(float);

  // h and h*r of all units, in chunks of 32 units: chunk c holds [RB][32] floats + 16 bytes of pad.
  // The 8 kg lanes of a warp read 8 different chunks (or half chunks) at the same offset; without
  // the pad that is an 8-way bank conflict on every load.  Where a lane's k range does not divide 32 (D = 192, 320,
  // 384, 448) a chunk is one lane's k range instead, so no float4 group straddles two chunks; the pad keeps the
  // 4 kg lanes of a load phase on distinct banks there too.
  constexpr int CH = 32 % KPG == 0 ? 32 : KPG, NCH = D / CH, SLOT = RB * CH + 4;
  __shared__ __align__(128) float hbuf[NCH][SLOT];
  __shared__ __align__(128) float hrbuf[NCH][SLOT];
  // state_to_state slice: [warp][q][lane][4 k] so a lane fetches four k of its column as one
  // vector; read in the candidate loop (the gate slice lives in registers for the whole sequence)
  extern __shared__ __align__(16) float w2s_dyn[];
  float (*w2s)[KQ][CPL2][32][4] = reinterpret_cast<float (*)[KQ][CPL2][32][4]>(w2s_dyn);
  // gate slice beyond the register-resident groups: [warp][q - QREG][j][lane][4 k], one float4 per lane and column
  // (the warp stride must be what ffma_smem_bytes allocates; QS = 1 only stands in for an empty slice)
  constexpr int QS = KQ > QREG ? KQ - QREG : 1;
  float (*w1s)[QS][CPL1][32][4] = reinterpret_cast<float (*)[QS][CPL1][32][4]>(w2s_dyn + (size_t)NWARP * KQ * CPL2 * 32 * 4);
  __shared__ __align__(8) unsigned long long mbar[2];   // [0]: h arrivals, [1]: h*r arrivals

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int kg = lane / CG, cg = lane % CG;
  const int cluster_id = blockIdx.x / CS;
  unsigned rank;
  asm volatile("mov.u32 %0, %%cluster_ctarank;\n" : "=r"(rank));
  const int dir = NDIR == 2 ? cluster_id & 1 : 0;                          // 0 forward, 1 backward
  const int row0 = (NDIR == 2 ? cluster_id >> 1 : cluster_id) * RB;       // first batch row of this cluster
  const int ul_warp = warp * NC2;             // first owned unit of this warp, local index
  const int u_warp = rank * UC + ul_warp;     // ... global unit index
  const int kpeer = (kg * KPG) / CH, koff = (kg * KPG) % CH;   // chunk and offset of this lane's k range

  const float* Wg = dir ? a.Wg_b : a.Wg_f;    // [D, 2D]  cols [update | reset]
  const float* Ws = dir ? a.Ws_b : a.Ws_f;    // [D, D]
  const float* h0 = dir ? a.h0_b : a.h0_f;    // [D]

  // ---- weights -> registers / shared memory (once) -----------------------------------
  // gate column cl of the warp (0..NC1): cl < NC2 -> update gate of unit u_warp + cl, else reset gate
  // pairs (k, k+1): the even-k and the odd-k partial sum of a column advance side by side (fma2) --
  // h arrives as (k, k+1) register pairs from the 16-byte loads anyway
  float2 w1[CPL1][QREG * 2];
#pragma unroll
  for (int j = 0; j < CPL1; ++j) {
    const int cl = cg * CPL1 + j;
    const int col = (cl < NC2) ? (u_warp + cl) : (D + u_warp + (cl - NC2));
#pragma unroll
    for (int kk = 0; kk < QREG * 2; ++kk)
      w1[j][kk] = make_float2(Wg[(long long)(kg * KPG + 2 * kk) * (2 * D) + col],
                              Wg[(long long)(kg * KPG + 2 * kk + 1) * (2 * D) + col]);
#pragma unroll
    for (int q = QREG; q < KQ; ++q)
#pragma unroll
      for (int i = 0; i < 4; ++i) w1s[warp][q - QREG][j][lane][i] = Wg[(long long)(kg * KPG + q * 4 + i) * (2 * D) + col];
  }
#pragma unroll
  for (int q = 0; q < KQ; ++q)
#pragma unroll
    for (int c2 = 0; c2 < CPL2; ++c2)
#pragma unroll
      for (int i = 0; i < 4; ++i)
        w2s[warp][q][c2][lane][i] = Ws[(long long)(kg * KPG + q * 4 + i) * D + u_warp + cg * CPL2 + c2];

  for (int i = tid; i < RB * D; i += NWARP * 32) {
    const int r = i / D, u = i % D;
    hbuf[u / CH][r * CH + u % CH] = h0[u];
  }

  // Lane roles after the reduce-scatters over the kg lanes (kg = lane >> 1, cg = lane & 1):
  //   gate sum      (row1 = kg >> 2, unit1 = kg & 3): update gate on cg 0 lanes, reset gate on cg 1 lanes
  //   candidate sum (row2 = kg >> 2, unit2 = cg * 2 + ((kg >> 1) & 1)), duplicated in the lane pair kg, kg ^ 1
  // h of (row, unit) lives in a register of lane 8 * row + 4 * (unit & 1) + (unit >> 1) (and its
  // duplicate); everything the epilogues need from other lanes comes by shuffle.
  static_assert(RB == 4 && NC2 == 4, "lane roles below assume 4 rows x 4 units per warp");
  const int row1 = kg >> 2, unit1 = kg & 3;
  const bool is_z = cg == 0;
  const int row2 = kg >> 2, unit2 = cg * 2 + ((kg >> 1) & 1);
  const int src_hold = 8 * row1 + 4 * (unit1 & 1) + (unit1 >> 1);          // h of my reset gate's unit
  const int src_z = (row2 * 4 + unit2) * 2;                                // update gate of my candidate's unit
  // sender role: lane = rowg * 8 + peer ships row rowg of this warp's 4 units to CTA `peer`
  const int rowg = lane >> 3, peer = lane & 7;
  const bool sender = peer < CS;
  const bool sender2 = peer + 8 < CS;   // clusters above 8 CTAs: lanes also ship to peer + 8
  int src_hr[4], src_h[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    src_hr[u] = (rowg * 4 + u) * 2 + 1;
    src_h[u] = 8 * rowg + 4 * (u & 1) + (u >> 1);
  }
  const uint32_t bar_h = smem_u32(&mbar[0]), bar_hr = smem_u32(&mbar[1]);
  // where this warp's 4 units of row rowg land in the receiver
  const uint32_t dst_h = map_to_rank(smem_u32(&hbuf[u_warp / CH][rowg * CH + u_warp % CH]), sender ? peer : 0);
  const uint32_t dst_hr = map_to_rank(smem_u32(&hrbuf[u_warp / CH][rowg * CH + u_warp % CH]), sender ? peer : 0);
  const uint32_t rbar_h = map_to_rank(bar_h, sender ? peer : 0), rbar_hr = map_to_rank(bar_hr, sender ? peer : 0);
  uint32_t dst_h2 = 0, dst_hr2 = 0, rbar_h2 = 0, rbar_hr2 = 0;
  if constexpr (CS > 8) {
    const int p2 = sender2 ? peer + 8 : 0;
    dst_h2 = map_to_rank(smem_u32(&hbuf[u_warp / CH][rowg * CH + u_warp % CH]), p2);
    dst_hr2 = map_to_rank(smem_u32(&hrbuf[u_warp / CH][rowg * CH + u_warp % CH]), p2);
    rbar_h2 = map_to_rank(bar_h, p2);
    rbar_hr2 = map_to_rank(bar_hr, p2);
  }
  if (tid == 0) {
    mbar_init(bar_h, 1);
    mbar_init(bar_hr, 1);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  float h_own = h0[u_warp + unit2];                                        // h(row2, unit2), same for every row at t = -1
  // training tape: broadcast initial state into its boundary slot of hext
  if constexpr (TAPE) {
    for (int i = tid; i < RB * UC; i += NWARP * 32) {
      const int r = i / UC, u = rank * UC + i % UC;
      if (row0 + r < a.B)
        a.hext[((long long)(dir ? a.T + 1 : 0) * a.B + row0 + r) * (NDIR * D) + dir * D + u] = h0[u];
    }
  }

  const int T = a.T, B = a.B;
  const long long pre_ld = 3LL * NDIR * D;                // [A | Gz | Gr] per direction
  const float* pre_dir = a.pre + (long long)dir * 3 * D;
  const int dt = dir ? -1 : 1;
  int t = dir ? (T - 1) : 0;
  // per-lane read pointers into the fork pre-activations, bumped by one time step per iteration
  const bool ok1 = row0 + row1 < B, ok2 = row0 + row2 < B;
  const float* pg_ptr = pre_dir + ((long long)t * B + row0 + row1) * pre_ld + (is_z ? D : 2 * D) + u_warp + unit1;
  const float* pa_ptr = pre_dir + ((long long)t * B + row0 + row2) * pre_ld + u_warp + unit2;
  const float* pm_ptr = a.mask ? a.mask + (long long)t * a.mask_tstride + row0 + row2 : nullptr;
  // tape slots of this lane's gate / candidate (same addresses the pre-activations are read from)
  float* tg_ptr = TAPE ? a.tape + (pg_ptr - a.pre) : nullptr;
  float* ta_ptr = TAPE ? a.tape + (pa_ptr - a.pre) : nullptr;
  const long long pre_step = (long long)dt * B * pre_ld, mask_step = (long long)dt * a.mask_tstride;
  float pg = 0.f, pa = 0.f, pm = 1.f;
  auto prefetch = [&]() {
    pg = ok1 ? __ldg(pg_ptr) : 0.f;
    pa = ok2 ? __ldg(pa_ptr) : 0.f;
    pm = (ok2 && pm_ptr) ? __ldg(pm_ptr) : 1.f;
    pg_ptr += pre_step; pa_ptr += pre_step;
    if (pm_ptr) pm_ptr += mask_step;
  };

  // every CTA of the cluster must be resident (and its mbarriers initialised) before any
  // remote copy is issued
  __syncthreads();
  cluster_sync_all();


  int sub_phase = dir ? ((T - 1) % a.subsample) : 0;   // t % subsample, maintained incrementally
  int t_out = t / a.subsample;
  prefetch();

  const bool tracer = g_bigru_trace_on && blockIdx.x == 0 && tid == 0;
  unsigned long long tr[6] = {0, 0, 0, 0, 0, 0};
  long long tc = 0;
#define BG_STAMP(j)                          \
  do {                                       \
    if (tracer) {                            \
      const long long now = clock64();       \
      tr[j] += (unsigned long long)(now - tc); \
      tc = now;                              \
    }                                        \
  } while (0)
  for (int s = 0; s < T; ++s, t += dt) {
    const float g_cur = pg, a_cur = pa, m_cur = pm;
    if (s + 1 < T) prefetch();
    if (tracer) tc = clock64();

    // h(s-1) from all peers has landed (step 0 uses the locally initialised h0)
    if (s > 0) mbar_wait(bar_h, (uint32_t)((s - 1) & 1));
    if (tid == 0) {
      mbar_arm(bar_h, FULL_BYTES);    // arrivals of h'(s)
      mbar_arm(bar_hr, FULL_BYTES);   // arrivals of (h*r)(s)
    }
    BG_STAMP(0);

    // ---- phase 1: gates of the owned units -----------------------------------------
    float acc1[N1];
    {
      float2 ap[N1];
#pragma unroll
      for (int i = 0; i < N1; ++i) ap[i] = make_float2(0.f, 0.f);
#pragma unroll
      for (int q = 0; q < QREG; ++q) {
#pragma unroll
        for (int r = 0; r < RB; ++r) {
          const float4 v = *reinterpret_cast<const float4*>(&hbuf[kpeer][r * CH + koff + q * 4]);
#pragma unroll
          for (int j = 0; j < CPL1; ++j) {
            float2 sacc = ap[r * CPL1 + j];
            sacc = fma2(make_float2(v.x, v.y), w1[j][q * 2 + 0], sacc);
            sacc = fma2(make_float2(v.z, v.w), w1[j][q * 2 + 1], sacc);
            ap[r * CPL1 + j] = sacc;
          }
        }
      }
#pragma unroll 1
      for (int q = QREG; q < KQ; ++q) {   // rolled: unrolled, the loads of later groups are hoisted and spill
        float4 w[CPL1];
#pragma unroll
        for (int j = 0; j < CPL1; ++j) w[j] = *reinterpret_cast<const float4*>(&w1s[warp][q - QREG][j][lane][0]);
#pragma unroll
        for (int r = 0; r < RB; ++r) {
          const float4 v = *reinterpret_cast<const float4*>(&hbuf[kpeer][r * CH + koff + q * 4]);
#pragma unroll
          for (int j = 0; j < CPL1; ++j) {
            float2 sacc = ap[r * CPL1 + j];
            sacc = fma2(make_float2(v.x, v.y), make_float2(w[j].x, w[j].y), sacc);
            sacc = fma2(make_float2(v.z, v.w), make_float2(w[j].z, w[j].w), sacc);
            ap[r * CPL1 + j] = sacc;
          }
        }
      }
#pragma unroll
      for (int i = 0; i < N1; ++i) acc1[i] = sum2(ap[i]);
    }
    BG_STAMP(1);
    warp_reduce_scatter<N1, CG>(acc1, lane);
    const float gate = fast_sigmoid(acc1[0] + g_cur);                    // z or r of (row1, unit1)
    if constexpr (TAPE) {
      if (ok1) *tg_ptr = gate;
      tg_ptr += pre_step;
    }
    const float hr_mine = __shfl_sync(0xffffffffu, h_own, src_hold) * gate;   // meaningful on reset-gate lanes
    {
      const float x = __shfl_sync(0xffffffffu, hr_mine, src_hr[0]), y = __shfl_sync(0xffffffffu, hr_mine, src_hr[1]);
      const float z = __shfl_sync(0xffffffffu, hr_mine, src_hr[2]), w = __shfl_sync(0xffffffffu, hr_mine, src_hr[3]);
      if (sender) st_async_v4(dst_hr, x, y, z, w, rbar_hr);
      if constexpr (CS > 8)
        if (sender2) st_async_v4(dst_hr2, x, y, z, w, rbar_hr2);
    }

    BG_STAMP(2);
    // ---- phase 2: candidate + blend for the owned units ----------------------------
    mbar_wait(bar_hr, (uint32_t)(s & 1));
    BG_STAMP(3);
    float acc2[N2];
    {
      float2 ap[N2];
#pragma unroll
      for (int i = 0; i < N2; ++i) ap[i] = make_float2(0.f, 0.f);
#pragma unroll
      for (int q = 0; q < KQ; ++q) {
        float4 w[CPL2];
#pragma unroll
        for (int c2 = 0; c2 < CPL2; ++c2) w[c2] = *reinterpret_cast<const float4*>(&w2s[warp][q][c2][lane][0]);
#pragma unroll
        for (int r = 0; r < RB; ++r) {
          const float4 v = *reinterpret_cast<const float4*>(&hrbuf[kpeer][r * CH + koff + q * 4]);
#pragma unroll
          for (int c2 = 0; c2 < CPL2; ++c2) {
            float2 sacc = ap[r * CPL2 + c2];
            sacc = fma2(make_float2(v.x, v.y), make_float2(w[c2].x, w[c2].y), sacc);
            sacc = fma2(make_float2(v.z, v.w), make_float2(w[c2].z, w[c2].w), sacc);
            ap[r * CPL2 + c2] = sacc;
          }
        }
      }
#pragma unroll
      for (int i = 0; i < N2; ++i) acc2[i] = sum2(ap[i]);
    }
    BG_STAMP(4);
    warp_reduce_scatter<N2, CG>(acc2, lane);
    {
      const float zg = __shfl_sync(0xffffffffu, gate, src_z);            // update gate of (row2, unit2)
      const float cand = fast_tanh(acc2[0] + a_cur);
      if constexpr (TAPE) {
        if (ok2 && (kg & 1) == 0) *ta_ptr = cand;       // the lane pair kg, kg ^ 1 holds the same value
        ta_ptr += pre_step;
      }
      float hn = cand * zg + h_own * (1.f - zg);
      hn = m_cur * hn + (1.f - m_cur) * h_own;
      h_own = hn;
      const float x = __shfl_sync(0xffffffffu, hn, src_h[0]), y = __shfl_sync(0xffffffffu, hn, src_h[1]);
      const float z = __shfl_sync(0xffffffffu, hn, src_h[2]), w = __shfl_sync(0xffffffffu, hn, src_h[3]);
      if (sender) st_async_v4(dst_h, x, y, z, w, rbar_h);
      if constexpr (CS > 8)
        if (sender2) st_async_v4(dst_h2, x, y, z, w, rbar_h2);
      if (sub_phase == 0 && peer == 0 && row0 + rowg < B)
        *reinterpret_cast<float4*>(a.out + ((long long)t_out * B + row0 + rowg) * (NDIR * D) + dir * D + u_warp) =
            make_float4(x, y, z, w);
      if (TAPE && peer == 0 && row0 + rowg < B)
        *reinterpret_cast<float4*>(a.hext + ((long long)(t + 1) * B + row0 + rowg) * (NDIR * D) + dir * D + u_warp) =
            make_float4(x, y, z, w);
    }
    BG_STAMP(5);
    // advance t % subsample and t / subsample without dividing
    if (dir == 0) {
      if (++sub_phase == a.subsample) { sub_phase = 0; ++t_out; }
    } else {
      if (sub_phase == 0) { sub_phase = a.subsample - 1; --t_out; } else { --sub_phase; }
    }
  }
#undef BG_STAMP
  if (tracer) {
#pragma unroll
    for (int j = 0; j < 6; ++j) g_bigru_trace[j] = tr[j];
    g_bigru_trace[6] = (unsigned long long)T;
  }
  // drain: the last h' copies must have landed everywhere before any CTA may exit
  mbar_wait(bar_h, (uint32_t)((T - 1) & 1));
  cluster_sync_all();
}

// dynamic shared memory of bigru_kernel<D, CS, NWARP, *>: the state_to_state slice, then the gate slice's groups beyond
// ffma_qreg
template <int D, int NWARP>
constexpr size_t ffma_smem_bytes() {
  return (size_t)NWARP * (D / 16 / 4) * 2 * 32 * 4 * sizeof(float) +
         (size_t)NWARP * (D / 64 - ffma_qreg<D>()) * 4 * 32 * 4 * sizeof(float);
}

// once per device: the dynamic shared memory, and clusters above 8 CTAs (D > 256) are non-portable
template <int D, int CS, int NDIR, int NWARP, bool TAPE>
int ffma_configure() {
  static bool configured[LVSR_MAX_DEVICES] = {false};
  const int dev = current_device();
  if (!configured[dev]) {
    LVSR_CUDA_OK(cudaFuncSetAttribute(bigru_kernel<D, CS, NDIR, NWARP, TAPE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)ffma_smem_bytes<D, NWARP>()));
    if (CS > 8)
      LVSR_CUDA_OK(cudaFuncSetAttribute(bigru_kernel<D, CS, NDIR, NWARP, TAPE>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    configured[dev] = true;
  }
  return 0;
}

// how many clusters of the FFMA kernel the device holds at once (0: none, the launch is refused)
template <int D, int CS, int NDIR, int NWARP, bool TAPE>
int ffma_clusters_resident() {
  static int per_dev[LVSR_MAX_DEVICES];
  static bool known[LVSR_MAX_DEVICES] = {false};
  const int dev = current_device();
  if (!known[dev]) {
    if (ffma_configure<D, CS, NDIR, NWARP, TAPE>()) return 0;
    known[dev] = true;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(CS * 64);
    cfg.blockDim = dim3(NWARP * 32);
    cfg.dynamicSmemBytes = ffma_smem_bytes<D, NWARP>();
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CS;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int k = 0;
    if (cudaOccupancyMaxActiveClusters(&k, bigru_kernel<D, CS, NDIR, NWARP, TAPE>, &cfg) != cudaSuccess) {
      cudaGetLastError();
      k = 0;
    }
    per_dev[dev] = k;
  }
  return per_dev[dev];
}

template <int D, int CS, int NDIR, int NWARP, bool TAPE>
int launch_bigru_t(const BiGruArgs& a, cudaStream_t stream, BiGruPlan* plan) {
  constexpr size_t W2S_BYTES = ffma_smem_bytes<D, NWARP>();
  if (int rc = ffma_configure<D, CS, NDIR, NWARP, TAPE>()) return rc;
  const int resident = ffma_clusters_resident<D, CS, NDIR, NWARP, TAPE>();
  if (resident <= 0)
    return set_error("bigru: this device holds no cluster of %d CTAs of the hidden-size-%d scan (%zu bytes of shared memory "
                     "each)", CS, D, W2S_BYTES);
  const int groups = ceil_div(a.B, RB);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(CS * groups * NDIR);
  cfg.blockDim = dim3(NWARP * 32);
  cfg.dynamicSmemBytes = W2S_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CS;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  static const bool trace = getenv("LVSR_BIGRU_TRACE") != nullptr;
  if (trace) {
    const int on = 1;
    LVSR_CUDA_OK(cudaMemcpyToSymbolAsync(g_bigru_trace_on, &on, sizeof(on), 0, cudaMemcpyHostToDevice, stream));
  }
  LVSR_CUDA_OK(cudaLaunchKernelEx(&cfg, bigru_kernel<D, CS, NDIR, NWARP, TAPE>, a));
  g_launch_count++;
  if (plan) *plan = {LVSR_ENC_BIGRU_FFMA, RB, CS, NDIR * groups, resident, ceil_div(NDIR * groups, resident)};
  if (trace) {
    unsigned long long h[8] = {0};
    LVSR_CUDA_OK(cudaMemcpyFromSymbolAsync(h, g_bigru_trace, sizeof(h), 0, cudaMemcpyDeviceToHost, stream));
    LVSR_CUDA_OK(cudaStreamSynchronize(stream));
    const double n = h[6] ? (double)h[6] : 1.0;
    fprintf(stderr,
            "[bigru trace] <%d,%d,%d> T=%llu cycles/step: wait_h=%.0f gates=%.0f gate_epi+send=%.0f wait_hr=%.0f "
            "cand=%.0f cand_epi+send=%.0f\n",
            D, CS, NWARP, h[6], h[0] / n, h[1] / n, h[2] / n, h[3] / n, h[4] / n, h[5] / n);
  }
  return 0;
}

// =====================================================================================================
// Tensor-core variant of the same scan (D = 256 at the metric batch): the two recurrent products run on
// mma.sync m16n8k16 (fp16 operands, fp32 accumulate) with the WEIGHT COLUMNS as the M dimension and the
// cluster's batch rows in the N = 8 slot: a CTA's 192 columns are 12 M tiles.  Up to the RB = 8 paragraph below this
// describes RB = 4.
//
// fp32 accuracy from fp16 operands: every operand is split into an fp16 head and an fp16 tail scaled by
// 2^11 (x = head + tail / 2048; both exact to ~2^-22 of x) and
//     head_w * head_h + (head_w * tail_h + tail_w * head_h) / 2048
// is accumulated in fp32 -- the error class of the 3xTF32 GEMMs with an m16n8k16 fp16 MMA covering twice the k of an
// m16n8k8 tf32 one.  It takes TWO MMAs per 16 k, not three: the
// N columns 0..3 of the B operand carry the heads of the four rows and the columns 4..7 their tails, so
// A = head_w yields head*head and head*tail in one instruction; the second one has A = tail_w.
// Weights are split once and stay in registers as ready-made A fragments (192 per lane).  h and h*r are split by the
// SENDER: the all-gather ships packed heads into one plane of the receiver's buffer and packed tails into another
// (4 bytes per unit in total, as fp32 would), so a B fragment is one 8-byte shared-memory load per k-step.  The
// fp32 state itself never leaves the registers of its owner threads: the split only feeds the products.
//
// Warp specialisation (12 warps, one CTA per SM; `setmaxnreg` moves registers from the elementwise warps to the MMA warps):
//   warps 4..11  MMA: one gate tile each over the full k, candidate tiles 4 x 2 k-halves; partial sums go to shared memory and
//                the warp ARRIVES on a named barrier -- it never waits for the elementwise work, only for operands
//                (mbarrier: all bytes of h / h*r have landed).
//   warps 0..3   elementwise: wait on the named barrier, add the partial sums + fork pre-activations, non-linearity,
//                split, one st.async per peer; every value is computed once or twice per CTA (the MUFU pipe is narrow).
//                Threads [0, 64) own (row, 4 units) and ship the heads, threads [64, 128) recompute the same values,
//                ship the tails and compute the update gate off the critical path.
// The exchange protocol is the FFMA kernel's (st.async + complete_tx on the receiver's mbarrier, no cluster barrier
// in the loop).
//
// RB = 8 rows per cluster (template parameter; halves the clusters of a batch, so a batch that would need two waves of
// 4-row clusters runs in one): the N = 8 slot carries the HEADS of the 8 rows and a second B fragment their TAILS, so a
// k-step issues three MMAs -- head_w * H_head, head_w * H_tail, tail_w * H_head -- into three accumulators of the same
// lane layout (tail * tail stays dropped, as for RB = 4).  A plane row interleaves each 4-unit group as
// [head01 head23 tail01 tail23]: one 16-byte load yields both B fragments of a k-step and one 16-byte st.async per peer
// ships heads and tails of a (row, 4 units) role.  The 128 elementwise threads own the 128 roles one each (r, z, the
// candidate and the sends of a role all run on its thread).
__device__ __forceinline__ void mma_f16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
constexpr float kTailScale = 2048.f, kTailUnscale = 1.f / 2048.f;
// (x, y) -> packed fp16 heads and packed scaled fp16 tails; the lower half of a word is the lower k index
__device__ __forceinline__ void split_pair(float x, float y, uint32_t& head, uint32_t& tail) {
  const __half2 h = __floats2half2_rn(x, y);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn((x - hf.x) * kTailScale, (y - hf.y) * kTailScale);
  head = *reinterpret_cast<const uint32_t*>(&h);
  tail = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ void st_async_v2_b32(uint32_t remote_addr, uint32_t x, uint32_t y, uint32_t remote_bar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v2.b32 [%0], {%1, %2}, [%3];\n" ::"r"(remote_addr),
               "r"(x), "r"(y), "r"(remote_bar)
               : "memory");
}
__device__ __forceinline__ void st_async_v4_b32(uint32_t remote_addr, uint4 v, uint32_t remote_bar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];\n" ::"r"(
                   remote_addr),
               "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"(remote_bar)
               : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;\n" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int count) {
  asm volatile("bar.arrive %0, %1;\n" ::"r"(id), "r"(count) : "memory");
}

constexpr int MMA_CS = 4, MMA_WARPS = 8, EW_WARPS = 4, MMA_THREADS = (MMA_WARPS + EW_WARPS) * 32;
// setmaxnreg redistributes the registers the CTA was LAUNCHED with (384 threads x 168), not the SM's whole file:
// 256 * 224 + 128 * 56 = 64512 = 384 * 168
constexpr int MMA_REGS = 224, EW_REGS = 56;
constexpr int PROGRESS_EVERY = 16;   // steps between two publications of BiGruArgs::progress

// Largest magnitude among the weights one warp turns into A fragments -> power-of-two scale that keeps the fp16 heads
// far inside the fp16 range (|w| * scale <= 2^14); the warp multiplies its partial sums by the inverse.  Parameters of
// any magnitude therefore give the same result as the fp32 kernel (1.0 / 1.0 for every sane model: an exact no-op).
__device__ __forceinline__ float range_scale(float warp_max_abs, float& inverse) {
  float scale = 1.f;
  inverse = 1.f;
  if (warp_max_abs > 16384.f && warp_max_abs < 3.0e38f) {
    const int e = ((__float_as_int(warp_max_abs) >> 23) & 0xff) - 127;   // 2^e <= max < 2^(e+1)
    scale = __int_as_float((127 - (e - 13)) << 23);                      // 2^-(e-13)
    inverse = __int_as_float((127 + (e - 13)) << 23);
  }
  return scale;
}

// NDIR as for bigru_kernel: 1 runs the forward direction in every cluster
template <int D, int NDIR, bool TAPE, int RB>
__global__ void __launch_bounds__(MMA_THREADS, 1)
bigru_mma_kernel(BiGruArgs a) {
  constexpr int CS = MMA_CS;
  constexpr int UC = D / CS;            // units owned by this CTA
  constexpr int MT1 = 2 * UC / 16;      // gate tiles: [z units | r units]
  constexpr int MT2 = UC / 16;          // candidate tiles
  constexpr int KS1 = MMA_WARPS / MT1;  // k splits of a gate tile over warps
  constexpr int KS2 = MMA_WARPS / MT2;
  constexpr int NK = D / 16;            // k-steps of a full product
  constexpr int NK1 = NK / KS1, NK2 = NK / KS2;
  constexpr int UG = UC / 4;            // 4-unit groups of this CTA
  constexpr int NROLE = RB * UG;        // (row, unit group) roles
  static_assert(MT1 * KS1 == MMA_WARPS && MT2 * KS2 == MMA_WARPS && NK1 * KS1 == NK && NK2 * KS2 == NK, "tile split");
  static_assert(NK1 % 2 == 0 && NK2 % 2 == 0, "two k-steps per round of the MMA loops");
  static_assert(RB == 4 || RB == 8, "N columns: 4 rows of heads + 4 rows of tails, or 8 rows of heads (and of tails)");
  static_assert((RB == 4 ? 2 : 1) * NROLE <= EW_WARPS * 32, "elementwise roles");
  // RB = 4: two planes [heads | tails], a plane row holds 2 words per 4-unit group = packed (u, u+1), (u+2, u+3); + 8
  // words: the 16 lanes of an 8-byte load phase (4 rows x 4 groups) then cover all 32 banks once.
  // RB = 8: one plane, a row holds 4 words per group = [head01 head23 tail01 tail23]; + 16 words: the 8 lanes of a
  // 16-byte load phase (2 rows x 4 groups) then cover all 32 banks once.
  constexpr int PLANES = RB == 4 ? 2 : 1;
  constexpr int RSH = RB == 4 ? D / 2 + 8 : D + 16;
  constexpr int RS1 = 2 * UC + 4, RS2 = UC + 4;   // 2 * RS mod 32 = 8: the row pairs of a C fragment spread over the banks
  constexpr uint32_t FULL_BYTES = RB * D * sizeof(uint32_t);

  __shared__ __align__(128) uint32_t hbuf[PLANES][RB][RSH];    // heads and tails of h
  __shared__ __align__(128) uint32_t hrbuf[PLANES][RB][RSH];   // ... of h * r
  __shared__ __align__(16) float red1[KS1][RB][RS1];
  __shared__ __align__(16) float red2[KS2][RB][RS2];
  __shared__ __align__(16) float zbuf[RB][UC];
  __shared__ __align__(8) unsigned long long mbar[2];
  __shared__ unsigned long long tr[12];   // section clocks of the two traced threads (only they touch them)

  const long long t_entry = clock64();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cluster_id = blockIdx.x / CS;
  unsigned rank;
  asm volatile("mov.u32 %0, %%cluster_ctarank;\n" : "=r"(rank));
  const int dir = NDIR == 2 ? cluster_id & 1 : 0;
  const int row0 = (NDIR == 2 ? cluster_id >> 1 : cluster_id) * RB;
  const float* h0 = dir ? a.h0_b : a.h0_f;
  const uint32_t bar_h = smem_u32(&mbar[0]), bar_hr = smem_u32(&mbar[1]);
  const int T = a.T, B = a.B;

  for (int i = tid; i < RB * D / 2; i += MMA_THREADS) {
    const int r = i / (D / 2), j = i % (D / 2);
    if constexpr (RB == 4)
      split_pair(h0[2 * j], h0[2 * j + 1], hbuf[0][r][j], hbuf[PLANES - 1][r][j]);
    else
      split_pair(h0[2 * j], h0[2 * j + 1], hbuf[0][r][4 * (j / 2) + j % 2], hbuf[0][r][4 * (j / 2) + 2 + j % 2]);
  }
  if (tid == 0) {
    mbar_init(bar_h, 1);
    mbar_init(bar_hr, 1);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    for (int j = 0; j < 12; ++j) tr[j] = 0;
  }
  // every CTA of the cluster must be resident (and its mbarriers initialised) before any remote copy is issued
  __syncthreads();
  cluster_sync_all();
  // a projection launched behind this scan as a programmatic dependent may start once every CTA of the scan runs: it
  // then only takes SMs this launch does not need
  asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory");
  const bool tracing = g_bigru_trace_on && blockIdx.x == 0;
  const long long t_loop = clock64();

  if (warp >= EW_WARPS) {
    // =================================== MMA warps ===================================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(MMA_REGS));
    const int g = lane >> 2, tq = lane & 3;
    const int m = warp - EW_WARPS;
    const int mt1 = m % MT1, kh = m / MT1;
    const int mt2 = m % MT2, kq = m / MT2;
    const float* Wg = dir ? a.Wg_b : a.Wg_f;
    const float* Ws = dir ? a.Ws_b : a.Ws_f;
    // ---- weights -> A fragments (once).  MMA k index kk of k-step ks <-> unit 16 ks + 4 (kk/2 % 4) + 2 (kk / 8) + kk % 2:
    // lane tq then needs the packed pairs of the four consecutive units 16 ks + 4 tq .. + 3 of a row = 8 bytes of a plane
    uint32_t wg_head[NK1][4], wg_tail[NK1][4], ws_head[NK2][4], ws_tail[NK2][4];
    float inv_g, inv_s;   // see range_scale()
    {
      float mx = 0.f;
#pragma unroll
      for (int j = 0; j < NK1; ++j)
#pragma unroll
        for (int half = 0; half < 2; ++half)
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const int ul = 16 * (mt1 % (MT1 / 2)) + g + 8 * half;
            const long long col = (mt1 < MT1 / 2 ? 0 : D) + rank * UC + ul;
            mx = fmaxf(mx, fabsf(Wg[(long long)((kh * NK1 + j) * 16 + 4 * tq + kk) * (2 * D) + col]));
          }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      const float sc = range_scale(mx, inv_g);
#pragma unroll
      for (int j = 0; j < NK1; ++j) {
        const int k0 = (kh * NK1 + j) * 16 + 4 * tq;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int ul = 16 * (mt1 % (MT1 / 2)) + g + 8 * half;
          const long long col = (mt1 < MT1 / 2 ? 0 : D) + rank * UC + ul;
          split_pair(sc * Wg[(long long)k0 * (2 * D) + col], sc * Wg[(long long)(k0 + 1) * (2 * D) + col], wg_head[j][half],
                     wg_tail[j][half]);
          split_pair(sc * Wg[(long long)(k0 + 2) * (2 * D) + col], sc * Wg[(long long)(k0 + 3) * (2 * D) + col],
                     wg_head[j][2 + half], wg_tail[j][2 + half]);
        }
      }
    }
    {
      float mx = 0.f;
#pragma unroll
      for (int j = 0; j < NK2; ++j)
#pragma unroll
        for (int half = 0; half < 2; ++half)
#pragma unroll
          for (int kk = 0; kk < 4; ++kk)
            mx = fmaxf(mx, fabsf(Ws[(long long)((kq * NK2 + j) * 16 + 4 * tq + kk) * D + rank * UC + 16 * mt2 + g + 8 * half]));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      const float sc = range_scale(mx, inv_s);
#pragma unroll
      for (int j = 0; j < NK2; ++j) {
        const int k0 = (kq * NK2 + j) * 16 + 4 * tq;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const long long col = rank * UC + 16 * mt2 + g + 8 * half;
          split_pair(sc * Ws[(long long)k0 * D + col], sc * Ws[(long long)(k0 + 1) * D + col], ws_head[j][half], ws_tail[j][half]);
          split_pair(sc * Ws[(long long)(k0 + 2) * D + col], sc * Ws[(long long)(k0 + 3) * D + col], ws_head[j][2 + half],
                     ws_tail[j][2 + half]);
        }
      }
    }
    // B fragments.  RB = 4: N column g < 4 = heads of batch row g, N column g >= 4 = tails of batch row g - 4 (one 8-byte
    // load per k-step).  RB = 8: N column g = batch row g, heads and tails of a k-step in one 16-byte load.
    const uint32_t* const hb = RB == 4 ? &hbuf[g / 4][g % 4][kh * NK1 * 8 + 2 * tq] : &hbuf[0][g][kh * NK1 * 16 + 4 * tq];
    const uint32_t* const hrb =
        RB == 4 ? &hrbuf[g / 4][g % 4][kq * NK2 * 8 + 2 * tq] : &hrbuf[0][g][kq * NK2 * 16 + 4 * tq];
    const uint2* hb2 = reinterpret_cast<const uint2*>(hb);
    const uint2* hrb2 = reinterpret_cast<const uint2*>(hrb);
    const uint4* hb4 = reinterpret_cast<const uint4*>(hb);
    const uint4* hrb4 = reinterpret_cast<const uint4*>(hrb);
    // C fragment rows: RB = 4 -> batch rows 2 (tq & 1) + {0, 1} (lanes tq < 2 store), RB = 8 -> 2 tq + {0, 1}
    float* const out1 = &red1[kh][RB == 4 ? 2 * (tq & 1) : 2 * tq][mt1 * 16 + g];
    float* const out2 = &red2[kq][RB == 4 ? 2 * (tq & 1) : 2 * tq][mt2 * 16 + g];
    const bool tracer = tracing && tid == EW_WARPS * 32;
#define BG_STAMP(j)                              \
  do {                                           \
    if (tracer) {                                \
      const unsigned long long now = clock64();  \
      tr[j] += now - tr[4];                      \
      tr[4] = now;                               \
    }                                            \
  } while (0)
    for (int s = 0; s < T; ++s) {
      if (tracer) tr[4] = clock64();
      if (s > 0) mbar_wait(bar_h, (uint32_t)((s - 1) & 1));
      if (tid == EW_WARPS * 32) {
        mbar_arm(bar_h, FULL_BYTES);    // arrivals of h'(s)
        mbar_arm(bar_hr, FULL_BYTES);   // arrivals of (h*r)(s)
      }
      BG_STAMP(0);
      if constexpr (RB == 8) {
        // three accumulation chains, one per product term; all three hold (weight column, batch row) in the same lanes.
        // (Splitting each into even / odd k-steps, as RB = 4 does, would reproduce its sums bit for bit but needs 12 more
        // registers than the MMA warps have.)
        float hh[4] = {0.f, 0.f, 0.f, 0.f}, ht[4] = {0.f, 0.f, 0.f, 0.f}, th[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int j = 0; j < NK1; ++j) {
          const uint4 v = hb4[j * 4];
          mma_f16(hh, wg_head[j], v.x, v.y);
          mma_f16(ht, wg_head[j], v.z, v.w);
          mma_f16(th, wg_tail[j], v.x, v.y);
        }
        out1[0] = (hh[0] + (ht[0] + th[0]) * kTailUnscale) * inv_g;
        out1[RS1] = (hh[1] + (ht[1] + th[1]) * kTailUnscale) * inv_g;
        out1[8] = (hh[2] + (ht[2] + th[2]) * kTailUnscale) * inv_g;
        out1[RS1 + 8] = (hh[3] + (ht[3] + th[3]) * kTailUnscale) * inv_g;
      } else {
        // four accumulation chains per warp (even / odd k-steps x head / tail weights): with two warps per scheduler a
        // chain of dependent MMAs would otherwise leave the tensor pipe waiting for its own results
        float c1[4] = {0.f, 0.f, 0.f, 0.f}, c2[4] = {0.f, 0.f, 0.f, 0.f};
        float d1[4] = {0.f, 0.f, 0.f, 0.f}, d2[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int j = 0; j < NK1; j += 2) {
          const uint2 v = hb2[j * 4], w = hb2[j * 4 + 4];
          mma_f16(c1, wg_head[j], v.x, v.y);
          mma_f16(c2, wg_tail[j], v.x, v.y);
          mma_f16(d1, wg_head[j + 1], w.x, w.y);
          mma_f16(d2, wg_tail[j + 1], w.x, w.y);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          c1[i] += d1[i];
          c2[i] += d2[i];
        }
        // lanes tq < 2 hold rows 2 tq, 2 tq + 1 of head*head (c1) and tail*head (c2); head*tail of the same rows
        // sits in c1 of lane + 2
#pragma unroll
        for (int i = 0; i < 4; ++i) c1[i] = (c1[i] + (__shfl_down_sync(0xffffffffu, c1[i], 2) + c2[i]) * kTailUnscale) * inv_g;
        if (tq < 2) {
          out1[0] = c1[0];
          out1[RS1] = c1[1];
          out1[8] = c1[2];
          out1[RS1 + 8] = c1[3];
        }
      }
      named_bar_arrive(1, MMA_THREADS);
      BG_STAMP(1);
      mbar_wait(bar_hr, (uint32_t)(s & 1));
      BG_STAMP(2);
      if constexpr (RB == 8) {
        float hh[4] = {0.f, 0.f, 0.f, 0.f}, ht[4] = {0.f, 0.f, 0.f, 0.f}, th[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int j = 0; j < NK2; ++j) {
          const uint4 v = hrb4[j * 4];
          mma_f16(hh, ws_head[j], v.x, v.y);
          mma_f16(ht, ws_head[j], v.z, v.w);
          mma_f16(th, ws_tail[j], v.x, v.y);
        }
        out2[0] = (hh[0] + (ht[0] + th[0]) * kTailUnscale) * inv_s;
        out2[RS2] = (hh[1] + (ht[1] + th[1]) * kTailUnscale) * inv_s;
        out2[8] = (hh[2] + (ht[2] + th[2]) * kTailUnscale) * inv_s;
        out2[RS2 + 8] = (hh[3] + (ht[3] + th[3]) * kTailUnscale) * inv_s;
      } else {
        float c1[4] = {0.f, 0.f, 0.f, 0.f}, c2[4] = {0.f, 0.f, 0.f, 0.f};
        float d1[4] = {0.f, 0.f, 0.f, 0.f}, d2[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int j = 0; j < NK2; j += 2) {
          const uint2 v = hrb2[j * 4], w = hrb2[j * 4 + 4];
          mma_f16(c1, ws_head[j], v.x, v.y);
          mma_f16(c2, ws_tail[j], v.x, v.y);
          mma_f16(d1, ws_head[j + 1], w.x, w.y);
          mma_f16(d2, ws_tail[j + 1], w.x, w.y);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          c1[i] += d1[i];
          c2[i] += d2[i];
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) c1[i] = (c1[i] + (__shfl_down_sync(0xffffffffu, c1[i], 2) + c2[i]) * kTailUnscale) * inv_s;
        if (tq < 2) {
          out2[0] = c1[0];
          out2[RS2] = c1[1];
          out2[8] = c1[2];
          out2[RS2 + 8] = c1[3];
        }
      }
      named_bar_arrive(2, MMA_THREADS);
      BG_STAMP(3);
    }
#undef BG_STAMP
    // drain: the last h' copies must have landed everywhere before any CTA may exit
    mbar_wait(bar_h, (uint32_t)((T - 1) & 1));
    if (g_bigru_trace_on && tid == EW_WARPS * 32 && blockIdx.x < 1024) {
      g_bigru_cta_cycles[0][blockIdx.x] = (unsigned long long)(t_loop - t_entry);
      g_bigru_cta_cycles[1][blockIdx.x] = (unsigned long long)(clock64() - t_loop);
    }
  } else {
    // =================================== elementwise warps ===========================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(EW_REGS));
    const bool active = tid < PLANES * NROLE;
    // RB = 4: the lead ships the heads and writes the outputs, its twin ships the tails and owns z.  RB = 8: one thread
    // per role does all of it
    const bool lead = tid < NROLE;
    const bool owns_z = RB == 8 || !lead;
    const int rid = tid % NROLE;
    const int ug = rid % UG, erow = active ? rid / UG : 0;
    const int u_loc = 4 * ug, u_glob = rank * UC + u_loc;
    const bool row_ok = active && row0 + erow < B;
    const bool writer = row_ok && lead;
    const int plane = RB == 4 && !lead ? 1 : 0;
    const int word = RB == 4 ? u_glob / 2 : u_glob;   // first word of this role's group in a plane row
    const uint32_t loc_h = smem_u32(&hbuf[plane][erow][word]), loc_hr = smem_u32(&hrbuf[plane][erow][word]);
    float h_own[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) h_own[i] = h0[u_glob + i];
    if constexpr (TAPE) {
      if (writer)
        *reinterpret_cast<float4*>(a.hext + ((long long)(dir ? T + 1 : 0) * B + row0 + erow) * (NDIR * D) + dir * D + u_glob) =
            make_float4(h_own[0], h_own[1], h_own[2], h_own[3]);
    }
    const long long pre_ld = 3LL * NDIR * D;
    const int dt = dir ? -1 : 1;
    int t = dir ? (T - 1) : 0;
    // fork pre-activations of this thread's 4 units: [inputs | update | reset]; every slot is re-loaded for the next step
    // right after its consumer, so a load has most of a step to land and nothing is double-buffered
    const long long pre_off = ((long long)t * B + row0 + erow) * pre_ld + (long long)dir * 3 * D + u_glob;
    const float* pre_ptr = a.pre + pre_off;
    float* tape_ptr = TAPE ? a.tape + pre_off : nullptr;
    const float* pm_ptr = a.mask ? a.mask + (long long)t * a.mask_tstride + row0 + erow : nullptr;
    const long long pre_step = (long long)dt * B * pre_ld, mask_step = (long long)dt * a.mask_tstride;
    const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 pa = zero4, pz = zero4, pr = zero4;
    float pm = 1.f;
    if (row_ok) {
      pa = __ldg(reinterpret_cast<const float4*>(pre_ptr));
      if (owns_z) pz = __ldg(reinterpret_cast<const float4*>(pre_ptr + D));
      pr = __ldg(reinterpret_cast<const float4*>(pre_ptr + 2 * D));
      if (pm_ptr) pm = __ldg(pm_ptr);
    }
    int sub_phase = dir ? ((T - 1) % a.subsample) : 0;   // t % subsample, maintained incrementally
    int t_out = t / a.subsample;
    const bool tracer = tracing && tid == 0;
#define BG_STAMP(j)                              \
  do {                                           \
    if (tracer) {                                \
      const unsigned long long now = clock64();  \
      tr[j] += now - tr[5];                      \
      tr[5] = now;                               \
    }                                            \
  } while (0)
    for (int s = 0; s < T; ++s, t += dt) {
      const bool more = s + 1 < T;
      if (tracer) tr[5] = clock64();
      named_bar_sync(1, MMA_THREADS);
      BG_STAMP(6);
      if (active) {
        float sr[4] = {pr.x, pr.y, pr.z, pr.w};
#pragma unroll
        for (int k = 0; k < KS1; ++k) {
          const float4 x = *reinterpret_cast<const float4*>(&red1[k][erow][UC + u_loc]);
          sr[0] += x.x; sr[1] += x.y; sr[2] += x.z; sr[3] += x.w;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) sr[i] = fast_sigmoid(sr[i]);
        uint32_t w0, w1, w2, w3;
        split_pair(h_own[0] * sr[0], h_own[1] * sr[1], w0, w1);
        split_pair(h_own[2] * sr[2], h_own[3] * sr[3], w2, w3);
        if constexpr (RB == 4) {
          const uint32_t x0 = lead ? w0 : w1, x1 = lead ? w2 : w3;
#pragma unroll
          for (int p = 0; p < CS; ++p) st_async_v2_b32(map_to_rank(loc_hr, p), x0, x1, map_to_rank(bar_hr, p));
        } else {
#pragma unroll
          for (int p = 0; p < CS; ++p) st_async_v4_b32(map_to_rank(loc_hr, p), make_uint4(w0, w2, w1, w3), map_to_rank(bar_hr, p));
        }
        if constexpr (TAPE) {
          if (writer) *reinterpret_cast<float4*>(tape_ptr + 2 * D) = make_float4(sr[0], sr[1], sr[2], sr[3]);
        }
        if (more && row_ok) pr = __ldg(reinterpret_cast<const float4*>(pre_ptr + pre_step + 2 * D));
        if (owns_z) {
          float sz[4] = {pz.x, pz.y, pz.z, pz.w};
#pragma unroll
          for (int k = 0; k < KS1; ++k) {
            const float4 x = *reinterpret_cast<const float4*>(&red1[k][erow][u_loc]);
            sz[0] += x.x; sz[1] += x.y; sz[2] += x.z; sz[3] += x.w;
          }
#pragma unroll
          for (int i = 0; i < 4; ++i) sz[i] = fast_sigmoid(sz[i]);
          *reinterpret_cast<float4*>(&zbuf[erow][u_loc]) = make_float4(sz[0], sz[1], sz[2], sz[3]);
          if constexpr (TAPE) {
            if (row_ok) *reinterpret_cast<float4*>(tape_ptr + D) = make_float4(sz[0], sz[1], sz[2], sz[3]);
          }
          if (more && row_ok) pz = __ldg(reinterpret_cast<const float4*>(pre_ptr + pre_step + D));
        }
      }
      BG_STAMP(7);
      named_bar_sync(2, MMA_THREADS);
      BG_STAMP(8);
      if (active) {
        float sc[4] = {pa.x, pa.y, pa.z, pa.w};
#pragma unroll
        for (int k = 0; k < KS2; ++k) {
          const float4 x = *reinterpret_cast<const float4*>(&red2[k][erow][u_loc]);
          sc[0] += x.x; sc[1] += x.y; sc[2] += x.z; sc[3] += x.w;
        }
        const float4 z4 = *reinterpret_cast<const float4*>(&zbuf[erow][u_loc]);
        const float zg[4] = {z4.x, z4.y, z4.z, z4.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          sc[i] = fast_tanh(sc[i]);
          float hn = sc[i] * zg[i] + h_own[i] * (1.f - zg[i]);
          hn = pm * hn + (1.f - pm) * h_own[i];
          h_own[i] = hn;
        }
        uint32_t w0, w1, w2, w3;
        split_pair(h_own[0], h_own[1], w0, w1);
        split_pair(h_own[2], h_own[3], w2, w3);
        if constexpr (RB == 4) {
          const uint32_t x0 = lead ? w0 : w1, x1 = lead ? w2 : w3;
#pragma unroll
          for (int p = 0; p < CS; ++p) st_async_v2_b32(map_to_rank(loc_h, p), x0, x1, map_to_rank(bar_h, p));
        } else {
#pragma unroll
          for (int p = 0; p < CS; ++p) st_async_v4_b32(map_to_rank(loc_h, p), make_uint4(w0, w2, w1, w3), map_to_rank(bar_h, p));
        }
        if (writer) {
          const float4 hv = make_float4(h_own[0], h_own[1], h_own[2], h_own[3]);
          if (sub_phase == 0)
            *reinterpret_cast<float4*>(a.out + ((long long)t_out * B + row0 + erow) * (NDIR * D) + dir * D + u_glob) = hv;
          if constexpr (TAPE) {
            *reinterpret_cast<float4*>(tape_ptr) = make_float4(sc[0], sc[1], sc[2], sc[3]);
            *reinterpret_cast<float4*>(a.hext + ((long long)(t + 1) * B + row0 + erow) * (NDIR * D) + dir * D + u_glob) = hv;
          }
        }
        pre_ptr += pre_step;
        if constexpr (TAPE) tape_ptr += pre_step;
        if (pm_ptr) pm_ptr += mask_step;
        if (more && row_ok) {
          pa = __ldg(reinterpret_cast<const float4*>(pre_ptr));
          if (pm_ptr) pm = __ldg(pm_ptr);
        }
      }
      // every PROGRESS_EVERY steps and after the last: the output stores of the elementwise warps so far are visible
      // at gpu scope, then one relaxed store says how many steps that covers (only these warps wait for it)
      if (a.progress && ((s % PROGRESS_EVERY) == PROGRESS_EVERY - 1 || !more)) {
        named_bar_sync(3, EW_WARPS * 32);
        if (tid == 0) {
          __threadfence();
          asm volatile("st.relaxed.gpu.global.b32 [%0], %1;\n" ::"l"(a.progress + blockIdx.x), "r"(s + 1) : "memory");
        }
      }
      BG_STAMP(9);
      // advance t % subsample and t / subsample without dividing
      if (dir == 0) {
        if (++sub_phase == a.subsample) { sub_phase = 0; ++t_out; }
      } else {
        if (sub_phase == 0) { sub_phase = a.subsample - 1; --t_out; } else { --sub_phase; }
      }
    }
#undef BG_STAMP
  }
  __syncthreads();
  if (tracing && tid == 0) {
#pragma unroll
    for (int j = 0; j < 4; ++j) g_bigru_trace[j] = tr[j];
#pragma unroll
    for (int j = 6; j < 10; ++j) g_bigru_trace[j - 2] = tr[j];
    g_bigru_trace[8] = (unsigned long long)T;
  }
  cluster_sync_all();
}

template <int D, int CS, int NWARP>
int launch_bigru(const BiGruArgs& a, cudaStream_t stream, BiGruPlan* plan) {
  LVSR_CHECK((a.tape == nullptr) == (a.hext == nullptr), "bigru: tape and hext go together");
  if (a.ndir == 1)
    return a.tape ? launch_bigru_t<D, CS, 1, NWARP, true>(a, stream, plan) : launch_bigru_t<D, CS, 1, NWARP, false>(a, stream, plan);
  return a.tape ? launch_bigru_t<D, CS, 2, NWARP, true>(a, stream, plan) : launch_bigru_t<D, CS, 2, NWARP, false>(a, stream, plan);
}

template <int D, bool TAPE>
int mma_launch_config(cudaLaunchConfig_t& cfg, cudaLaunchAttribute* attr, int clusters, cudaStream_t stream) {
  cfg = {};
  cfg.gridDim = dim3(MMA_CS * clusters);
  cfg.blockDim = dim3(MMA_THREADS);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = stream;
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = MMA_CS;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return 0;
}

// how many clusters of the tensor-core kernel the device holds at once (one CTA per SM, 4 SMs of one GPC per cluster)
template <int D, int NDIR, int RB>
int mma_clusters_resident() {
  static int per_dev[LVSR_MAX_DEVICES];
  static bool known[LVSR_MAX_DEVICES] = {false};
  const int dev = current_device();
  if (!known[dev]) {
    known[dev] = true;
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attr[1];
    int k = 0;
    if (mma_launch_config<D, false>(cfg, attr, 64, nullptr) != 0 ||
        cudaOccupancyMaxActiveClusters(&k, bigru_mma_kernel<D, NDIR, false, RB>, &cfg) != cudaSuccess) {
      cudaGetLastError();
      k = 0;
    }
    per_dev[dev] = k;
  }
  return per_dev[dev];
}

// waves of a launch of B rows: clusters never talk to each other, so a launch with more clusters than the device holds
// at once runs them in turns, and every wave costs a whole sequence of steps (0: the kernel cannot be resident at all)
template <int D, int NDIR, int RB>
int mma_waves(int B) {
  const int resident = mma_clusters_resident<D, NDIR, RB>();
  return resident > 0 ? ceil_div(NDIR * ceil_div(B, RB), resident) : 0;
}

template <int D, int NDIR, bool TAPE, int RB>
int launch_bigru_mma_t(const BiGruArgs& a, cudaStream_t stream) {
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  const int clusters = ceil_div(a.B, RB) * NDIR;
  if (int rc = mma_launch_config<D, TAPE>(cfg, attr, clusters, stream)) return rc;
  static const bool trace = getenv("LVSR_BIGRU_TRACE") != nullptr;
  if (trace) {
    const int on = 1;
    LVSR_CUDA_OK(cudaMemcpyToSymbolAsync(g_bigru_trace_on, &on, sizeof(on), 0, cudaMemcpyHostToDevice, stream));
  }
  LVSR_CUDA_OK(cudaLaunchKernelEx(&cfg, bigru_mma_kernel<D, NDIR, TAPE, RB>, a));
  g_launch_count++;
  if (trace) {
    unsigned long long h[12] = {0};
    LVSR_CUDA_OK(cudaMemcpyFromSymbolAsync(h, g_bigru_trace, sizeof(h), 0, cudaMemcpyDeviceToHost, stream));
    LVSR_CUDA_OK(cudaStreamSynchronize(stream));
    const double n = h[8] ? (double)h[8] : 1.0;
    fprintf(stderr, "[bigru trace] mma<%d> RB=%d B=%d clusters=%d resident=%d waves=%d\n", D, RB, a.B, clusters,
            mma_clusters_resident<D, NDIR, RB>(), mma_waves<D, NDIR, RB>(a.B));
    fprintf(stderr,
            "[bigru trace] mma<%d> T=%llu cycles/step  MMA warp: wait_h=%.0f gates=%.0f wait_hr=%.0f cand=%.0f | elementwise: "
            "wait_gates=%.0f r+send(+z)=%.0f wait_cand=%.0f cand+send+stores=%.0f\n",
            D, h[8], h[0] / n, h[1] / n, h[2] / n, h[3] / n, h[4] / n, h[5] / n, h[6] / n, h[7] / n);
    static unsigned long long cc[2][1024];
    LVSR_CUDA_OK(cudaMemcpyFromSymbol(cc, g_bigru_cta_cycles, sizeof(cc)));
    const int nc = (int)cfg.gridDim.x < 1024 ? (int)cfg.gridDim.x : 1024;
    for (int w = 0; w < 2; ++w) {
      unsigned long long lo = ~0ull, hi = 0;
      double sum = 0;
      for (int c = 0; c < nc; ++c) {
        lo = cc[w][c] < lo ? cc[w][c] : lo;
        hi = cc[w][c] > hi ? cc[w][c] : hi;
        sum += (double)cc[w][c];
      }
      fprintf(stderr, "[bigru trace]   %s cycles per CTA: min %llu avg %.0f max %llu%s\n", w ? "loop" : "entry->loop", lo, sum / nc, hi,
              w ? "" : "");
    }
    fprintf(stderr, "[bigru trace]   loop cycles per step, slowest CTA: %.0f\n", 0.0 + (double)[&] { unsigned long long m = 0; for (int c = 0; c < nc; ++c) m = cc[1][c] > m ? cc[1][c] : m; return m; }() / n);
  }
  return 0;
}

template <int D, int NDIR, int RB>
int launch_bigru_mma(const BiGruArgs& a, cudaStream_t stream, BiGruPlan* plan) {
  LVSR_CHECK((a.tape == nullptr) == (a.hext == nullptr), "bigru: tape and hext go together");
  if (int rc = a.tape ? launch_bigru_mma_t<D, NDIR, true, RB>(a, stream) : launch_bigru_mma_t<D, NDIR, false, RB>(a, stream))
    return rc;
  if (plan)
    *plan = {LVSR_ENC_BIGRU_MMA, RB, MMA_CS, ceil_div(a.B, RB) * NDIR, mma_clusters_resident<D, NDIR, RB>(),
             mma_waves<D, NDIR, RB>(a.B)};
  return 0;
}

// the tensor-core plan of a batch of B rows with NDIR directions: RB 4, or 8 where that saves a wave (see bigru_plan)
template <int NDIR>
int mma_plan(int B, BiGruPlan* plan) {
  // 8-row clusters cost a third MMA per k-step and twice the elementwise work of a step, but halve the clusters:
  // worth it only where that saves a wave
  int rb = 4;
  const int w8 = mma_waves<256, NDIR, 8>(B);
  if (w8 > 0 && w8 < mma_waves<256, NDIR, 4>(B)) rb = 8;
  if (const char* e = getenv("LVSR_BIGRU_RB")) {
    rb = atoi(e);
    if (rb != 4 && rb != 8) return set_error("bigru: LVSR_BIGRU_RB=%s (expected 4 or 8)", e);
  }
  const int clusters = ceil_div(B, rb) * NDIR;
  *plan = rb == 8 ? BiGruPlan{LVSR_ENC_BIGRU_MMA, 8, MMA_CS, clusters, mma_clusters_resident<256, NDIR, 8>(),
                              mma_waves<256, NDIR, 8>(B)}
                  : BiGruPlan{LVSR_ENC_BIGRU_MMA, 4, MMA_CS, clusters, mma_clusters_resident<256, NDIR, 4>(),
                              mma_waves<256, NDIR, 4>(B)};
  return 0;
}

}  // namespace

bool bigru_supported(int D) { return D >= 64 && D <= 512 && D % 64 == 0; }

int bigru_plan(const BiGruArgs& a, BiGruPlan* plan) {
  *plan = {};
  if (a.T <= 0 || a.B <= 0) return 0;
  LVSR_CHECK(a.ndir == 1 || a.ndir == 2, "bigru: %d directions (1 or 2)", a.ndir);
  // hidden size 256: tensor-core products.  Clusters never talk to each other, so a batch with more clusters than the
  // device holds at once (mma_clusters_resident, from the occupancy query) simply runs in waves -- still
  // ahead of the FFMA kernels, which would have to put two or more CTAs on every SM for such a batch.
  bool mma = a.D == 256 && (a.ndir == 1 ? mma_clusters_resident<256, 1, 4>() : mma_clusters_resident<256, 2, 4>()) > 0;
  if (const char* e = getenv("LVSR_BIGRU_MMA")) mma = a.D == 256 && atoi(e) != 0;
  if (mma) return a.ndir == 1 ? mma_plan<1>(a.B, plan) : mma_plan<2>(a.B, plan);
  LVSR_CHECK(bigru_supported(a.D), "bigru: unsupported hidden size %d (supported: multiples of 64 from 64 to 512)", a.D);
  // the FFMA kernel's occupancy (resident, waves) is queried when it is launched
  *plan = {LVSR_ENC_BIGRU_FFMA, RB, a.D / 32, a.ndir * ceil_div(a.B, RB), 0, 0};
  return 0;
}

// The FFMA kernel publishes no progress (BiGruArgs::progress is for the tensor-core kernel only).
int bigru_layer(const BiGruArgs& a, cudaStream_t stream, BiGruPlan* plan) {
  BiGruPlan pl;
  if (plan) *plan = {};
  if (int rc = bigru_plan(a, &pl)) return rc;
  if (a.T <= 0 || a.B <= 0) return 0;
  if (pl.kernel == LVSR_ENC_BIGRU_MMA) {
    if (a.ndir == 1) return pl.rb == 8 ? launch_bigru_mma<256, 1, 8>(a, stream, plan) : launch_bigru_mma<256, 1, 4>(a, stream, plan);
    return pl.rb == 8 ? launch_bigru_mma<256, 2, 8>(a, stream, plan) : launch_bigru_mma<256, 2, 4>(a, stream, plan);
  }
  switch (a.D) {
    case 64: return launch_bigru<64, 2, 8>(a, stream, plan);
    case 128: return launch_bigru<128, 4, 8>(a, stream, plan);
    case 192: return launch_bigru<192, 6, 8>(a, stream, plan);
    case 256: return launch_bigru<256, 8, 8>(a, stream, plan);
    case 320: return launch_bigru<320, 10, 8>(a, stream, plan);
    case 384: return launch_bigru<384, 12, 8>(a, stream, plan);
    case 448: return launch_bigru<448, 14, 8>(a, stream, plan);
    default: return launch_bigru<512, 16, 8>(a, stream, plan);
  }
}

}  // namespace lvsr
