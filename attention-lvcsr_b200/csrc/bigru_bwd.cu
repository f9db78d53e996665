// Backward pass (BPTT) of one bidirectional GatedRecurrent layer: one persistent, cluster-resident
// kernel for BOTH directions -- the reverse-time twin of bigru.cu.
//
// What it differentiates (B/bricks/recurrent.py:608-620, the scan of :224-231 run backwards):
//     g = sigma(h W_g + G_t) ; z = g[:, :D] ; r = g[:, D:]
//     c = tanh((h * r) W_s + A_t) ; h~ = c z + h (1 - z) ; h' = m h~ + (1 - m) h
// Given dL/dh' (from the layer output and from the later step) one step yields
//     dh~ = m dh' ; dc = dh~ z ; dz = dh~ (c - h)
//     dA  = dc (1 - c^2)                                   -> gradient of fork_inputs pre-activation
//     d(hr) = dA W_s^T ; dr = d(hr) h ; dGz = dz z (1-z) ; dGr = dr r (1-r)   -> fork_gate_inputs
//     dh  = (1-m) dh' + dh~ (1-z) + d(hr) r + [dGz | dGr] W_g^T
// i.e. again two DEPENDENT skinny products per step, now with the transposed weights.  The weight
// gradients are NOT accumulated here: the kernel leaves dA, dGz, dGr (in place over the forward's
// saved c, z, r) and h*r for every step, and the caller turns them into four large GEMMs
// (dW_fork = X^T dPre, dX = dPre W_fork^T, dW_s = (h*r)^T dA, dW_g = H_prev^T [dGz|dGr]).
//
// Mapping: a cluster of CS CTAs owns RB = 4 batch rows of one direction, CTA `rank` owns 32
// hidden units.  Per step the owned dA (then [dGz|dGr]) of all 4 rows travel as ONE 16-byte
// `st.async` per unit and peer into the receivers' shared memory, crediting the receiver's
// mbarrier -- the all-gather machinery of the forward kernel.  W_s^T slice in registers, W_g^T
// slice in shared memory (k-major, padded so the 8 k-groups of a warp hit distinct banks);
// thread = (k-group 0..7, unit), 4 rows per thread, cross-k reduction by shuffles.
// Every D = 64, 128, ..., 512 runs, with CS = D / 32 (clusters above 8 CTAs are non-portable); from D = 384 on the
// shared memory leaves room for one CTA per SM.  NDIR = 1 is the layer of a forward-only encoder (net.bidir False):
// every cluster runs the forward direction and the tape, hext, dout and hr_out hold one direction.
#include "kernels.h"

namespace lvsr {

namespace {

constexpr int RB = 4;
constexpr int UC = 32;          // units per CTA
constexpr int NT = 256;
constexpr int WSTR = UC + 4;    // shared-memory row stride of the k-major weight slices

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
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
__device__ __forceinline__ void st_async_v4(uint32_t remote_addr, float4 v, uint32_t remote_bar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1, %2, %3, %4}, [%5];\n" ::"r"(
                   remote_addr),
               "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "r"(remote_bar)
               : "memory");
}

__host__ __device__ constexpr size_t bwd_smem_bytes(int D) {
  return ((size_t)2 * D * WSTR) * sizeof(float) + ((size_t)3 * D + 2 * UC) * sizeof(float4);
}
// CTAs per SM the shared memory allows (228 KB per SM, 1 KB of it reserved per CTA); the register budget follows it, so
// the wide layers, which hold one CTA per SM anyway, get the registers that keep them from spilling
__host__ __device__ constexpr int bwd_min_blocks(int D) { return 2 * (bwd_smem_bytes(D) + 1024) <= 228 * 1024 ? 2 : 1; }

template <int D, int CS, int NDIR>
__global__ void __launch_bounds__(NT, bwd_min_blocks(D)) bigru_bwd_kernel(BiGruBwdArgs a) {
  static_assert(D == CS * UC, "32 units per CTA");
  static_assert(NDIR == 1 || NDIR == 2, "one or two directions");
  constexpr int KA = D / 8;         // k values per thread, first product  (K = D)
  constexpr int KB = 2 * D / 8;     // second product (K = 2D)
  extern __shared__ __align__(16) float smem[];
  float* WtB = smem;                                   // [2D][WSTR]: W_g[j, c] at [c][j]
  float4* bufA = reinterpret_cast<float4*>(smem + (size_t)2 * D * WSTR);   // [D]  dA of all units, 4 rows each
  float4* bufB = bufA + D;                             // [2D] dGz | dGr
  float4* red1 = bufB + 2 * D;                         // [UC]
  float4* red2 = red1 + UC;                            // [UC]
  __shared__ __align__(8) unsigned long long mbar[2];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int jj = lane & 3, ks = lane >> 2, j = warp * 4 + jj;        // product role: unit j, k-group ks
  const int cluster_id = blockIdx.x / CS;
  unsigned rank;
  asm volatile("mov.u32 %0, %%cluster_ctarank;\n" : "=r"(rank));
  const int dir = NDIR == 2 ? cluster_id & 1 : 0;
  const int row0 = (NDIR == 2 ? cluster_id >> 1 : cluster_id) * RB;
  const int u0 = rank * UC;
  const float* Wg = dir ? a.Wg_b : a.Wg_f;
  const float* Ws = dir ? a.Ws_b : a.Ws_f;
  const int T = a.T, B = a.B;

  // ---- weights: W_s^T slice -> registers, W_g^T slice -> shared memory (once) ----------------
  float wA[KA];
#pragma unroll
  for (int kk = 0; kk < KA; ++kk) wA[kk] = Ws[(long long)(u0 + j) * D + kk * 8 + ks];
  for (int i = tid; i < UC * 2 * D; i += NT) {
    const int jl = i / (2 * D), c = i % (2 * D);
    WtB[(size_t)c * WSTR + jl] = Wg[(long long)(u0 + jl) * (2 * D) + c];
  }
  const uint32_t barA = smem_u32(&mbar[0]), barB = smem_u32(&mbar[1]);
  if (tid == 0) {
    mbar_init(barA, 1);
    mbar_init(barB, 1);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();
  cluster_sync_all();

  // ---- element-wise owner: warp 0, lane = owned unit, all RB rows in registers ---------------
  const int ju = u0 + lane;                                 // global unit of this lane (warp 0)
  const long long pre_ld = 3LL * NDIR * D;
  const int dt = dir ? 1 : -1;                              // backward in the scan's own order
  int t = dir ? 0 : T - 1;
  float dh[RB] = {0.f, 0.f, 0.f, 0.f};
  float nz[RB], nr[RB], nc[RB], nh[RB], nm[RB], ng[RB];      // prefetched operands of the coming step
  auto prefetch = [&](int tt) {
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      const int row = row0 + r;
      nz[r] = nr[r] = nc[r] = nh[r] = ng[r] = 0.f;
      nm[r] = 1.f;
      if (row < B) {
        const float* tp = a.tape + ((long long)tt * B + row) * pre_ld + (long long)dir * 3 * D;
        nc[r] = __ldg(tp + ju); nz[r] = __ldg(tp + D + ju); nr[r] = __ldg(tp + 2 * D + ju);
        // h_prev: forward direction = state after time tt-1 (slot tt), backward = after tt+1 (slot tt+2)
        nh[r] = __ldg(a.hext + ((long long)(dir ? tt + 2 : tt) * B + row) * (NDIR * D) + dir * D + ju);
        if (a.mask) nm[r] = __ldg(a.mask + (long long)tt * a.mask_tstride + row);
        if (tt % a.subsample == 0)
          ng[r] = __ldg(a.dout + ((long long)(tt / a.subsample) * B + row) * (NDIR * D) + dir * D + ju);
      }
    }
  };
  if (warp == 0) prefetch(t);

  // remote addresses: held in registers at CS = 2, 4 and 8 (as the kernel always did); at the other sizes 5 * CS of them
  // would spill, and `mapa` in the loop is cheap
  constexpr bool REMOTE_REGS = CS <= 4 || CS == 8;
  constexpr int NR = REMOTE_REGS ? CS : 1;
  uint32_t dstA[NR], dstB0[NR], dstB1[NR], rbarA[NR], rbarB[NR];
#pragma unroll
  for (int p = 0; p < NR; ++p) {
    dstA[p] = map_to_rank(smem_u32(&bufA[ju]), p);
    dstB0[p] = map_to_rank(smem_u32(&bufB[ju]), p);
    dstB1[p] = map_to_rank(smem_u32(&bufB[D + ju]), p);
    rbarA[p] = map_to_rank(barA, p);
    rbarB[p] = map_to_rank(barB, p);
  }

  for (int s = 0; s < T; ++s, t += dt) {
    float z[RB], r[RB], c[RB], h[RB], keep[RB], daz[RB];
    if (tid == 0) {
      mbar_arm(barA, (uint32_t)(D * sizeof(float4)));
      mbar_arm(barB, (uint32_t)(2 * D * sizeof(float4)));
    }
    if (warp == 0) {
      float dac[RB];
#pragma unroll
      for (int q = 0; q < RB; ++q) {
        z[q] = nz[q]; r[q] = nr[q]; c[q] = nc[q]; h[q] = nh[q];
        const float tot = dh[q] + ng[q];
        const float dht = nm[q] * tot;
        keep[q] = (1.f - nm[q]) * tot + dht * (1.f - z[q]);
        const float dc = dht * z[q], dz = dht * (c[q] - h[q]);
        dac[q] = dc * (1.f - c[q] * c[q]);
        daz[q] = dz * z[q] * (1.f - z[q]);
      }
      const float4 v = make_float4(dac[0], dac[1], dac[2], dac[3]);
      if constexpr (REMOTE_REGS) {
#pragma unroll
        for (int p = 0; p < CS; ++p) st_async_v4(dstA[p], v, rbarA[p]);
      } else {
#pragma unroll
        for (int p = 0; p < CS; ++p) st_async_v4(map_to_rank(smem_u32(&bufA[ju]), p), v, map_to_rank(barA, p));
      }
      // dA of this step: in place over the saved candidate
#pragma unroll
      for (int q = 0; q < RB; ++q)
        if (row0 + q < B) a.tape[((long long)t * B + row0 + q) * pre_ld + (long long)dir * 3 * D + ju] = dac[q];
      if (s + 1 < T) prefetch(t + dt);
    }
    // ---- product 1: d(hr)[owned j] = sum_u dA[u] W_s[j, u] -------------------------------------
    mbar_wait(barA, (uint32_t)(s & 1));
    {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int kk = 0; kk < KA; ++kk) {
        const float4 x = bufA[kk * 8 + ks];
        const float w = wA[kk];
        acc.x = fmaf(x.x, w, acc.x); acc.y = fmaf(x.y, w, acc.y); acc.z = fmaf(x.z, w, acc.z); acc.w = fmaf(x.w, w, acc.w);
      }
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o); acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
        acc.z += __shfl_xor_sync(0xffffffffu, acc.z, o); acc.w += __shfl_xor_sync(0xffffffffu, acc.w, o);
      }
      if (ks == 0) red1[j] = acc;
    }
    __syncthreads();
    if (warp == 0) {
      const float4 d4 = red1[lane];
      const float dhr[RB] = {d4.x, d4.y, d4.z, d4.w};
      float dar[RB], hr[RB];
#pragma unroll
      for (int q = 0; q < RB; ++q) {
        const float dr = dhr[q] * h[q];
        keep[q] += dhr[q] * r[q];
        dar[q] = dr * r[q] * (1.f - r[q]);
        hr[q] = h[q] * r[q];
      }
      const float4 vz = make_float4(daz[0], daz[1], daz[2], daz[3]), vr = make_float4(dar[0], dar[1], dar[2], dar[3]);
      if constexpr (REMOTE_REGS) {
#pragma unroll
        for (int p = 0; p < CS; ++p) {
          st_async_v4(dstB0[p], vz, rbarB[p]);
          st_async_v4(dstB1[p], vr, rbarB[p]);
        }
      } else {
#pragma unroll
        for (int p = 0; p < CS; ++p) {
          const uint32_t rbar = map_to_rank(barB, p);
          st_async_v4(map_to_rank(smem_u32(&bufB[ju]), p), vz, rbar);
          st_async_v4(map_to_rank(smem_u32(&bufB[D + ju]), p), vr, rbar);
        }
      }
#pragma unroll
      for (int q = 0; q < RB; ++q) {
        if (row0 + q < B) {
          float* tp = a.tape + ((long long)t * B + row0 + q) * pre_ld + (long long)dir * 3 * D;
          tp[D + ju] = daz[q];
          tp[2 * D + ju] = dar[q];
          a.hr_out[((long long)t * B + row0 + q) * (NDIR * D) + dir * D + ju] = hr[q];
        }
      }
    }
    // ---- product 2: dh[owned j] += sum_c [dGz|dGr][c] W_g[j, c] ---------------------------------
    mbar_wait(barB, (uint32_t)(s & 1));
    {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 8
      for (int kk = 0; kk < KB; ++kk) {
        const int cidx = kk * 8 + ks;
        const float4 x = bufB[cidx];
        const float w = WtB[(size_t)cidx * WSTR + j];
        acc.x = fmaf(x.x, w, acc.x); acc.y = fmaf(x.y, w, acc.y); acc.z = fmaf(x.z, w, acc.z); acc.w = fmaf(x.w, w, acc.w);
      }
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o); acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
        acc.z += __shfl_xor_sync(0xffffffffu, acc.z, o); acc.w += __shfl_xor_sync(0xffffffffu, acc.w, o);
      }
      if (ks == 0) red2[j] = acc;
    }
    __syncthreads();
    if (warp == 0) {
      const float4 d4 = red2[lane];
      dh[0] = keep[0] + d4.x; dh[1] = keep[1] + d4.y; dh[2] = keep[2] + d4.z; dh[3] = keep[3] + d4.w;
    }
  }
  // gradient with respect to the (broadcast) initial state of this direction
  if (warp == 0) {
#pragma unroll
    for (int q = 0; q < RB; ++q)
      if (row0 + q < B) a.dh0[((long long)dir * B + row0 + q) * D + ju] = dh[q];
  }
  cluster_sync_all();   // no CTA exits while a peer may still address its shared memory
}

template <int D, int CS, int NDIR>
int launch_bwd(const BiGruBwdArgs& a, cudaStream_t stream) {
  constexpr size_t SMEM = bwd_smem_bytes(D);
  static bool configured[LVSR_MAX_DEVICES] = {false};
  static int resident[LVSR_MAX_DEVICES];
  const int dev = current_device();
  const int groups = ceil_div(a.B, RB);
  cudaLaunchConfig_t cfg = {};
  if (!configured[dev]) {
    LVSR_CUDA_OK(cudaFuncSetAttribute(bigru_bwd_kernel<D, CS, NDIR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM));
    if (CS > 8) LVSR_CUDA_OK(cudaFuncSetAttribute(bigru_bwd_kernel<D, CS, NDIR>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    configured[dev] = true;
    resident[dev] = -1;
  }
  cfg.gridDim = dim3(CS * groups * NDIR);
  cfg.blockDim = dim3(NT);
  cfg.dynamicSmemBytes = SMEM;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CS;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (resident[dev] < 0) {
    int k = 0;
    if (cudaOccupancyMaxActiveClusters(&k, bigru_bwd_kernel<D, CS, NDIR>, &cfg) != cudaSuccess) {
      cudaGetLastError();
      k = 0;
    }
    resident[dev] = k;
  }
  if (resident[dev] <= 0)
    return set_error("bigru backward: this device holds no cluster of %d CTAs of the hidden-size-%d scan (%zu bytes of "
                     "shared memory each)", CS, D, SMEM);
  LVSR_CUDA_OK(cudaLaunchKernelEx(&cfg, bigru_bwd_kernel<D, CS, NDIR>, a));
  g_launch_count++;
  return 0;
}

template <int NDIR>
int launch_bwd_width(const BiGruBwdArgs& a, cudaStream_t stream) {
  switch (a.D) {
    case 64: return launch_bwd<64, 2, NDIR>(a, stream);
    case 128: return launch_bwd<128, 4, NDIR>(a, stream);
    case 192: return launch_bwd<192, 6, NDIR>(a, stream);
    case 256: return launch_bwd<256, 8, NDIR>(a, stream);
    case 320: return launch_bwd<320, 10, NDIR>(a, stream);
    case 384: return launch_bwd<384, 12, NDIR>(a, stream);
    case 448: return launch_bwd<448, 14, NDIR>(a, stream);
    case 512: return launch_bwd<512, 16, NDIR>(a, stream);
    default:
      return set_error("bigru backward: unsupported hidden size %d (supported: multiples of 64 from 64 to 512)", a.D);
  }
}

}  // namespace

int bigru_layer_backward(const BiGruBwdArgs& a, cudaStream_t stream, int* cs_out) {
  ProfScope prof("bigru_bwd", stream);
  if (cs_out) *cs_out = 0;
  if (a.T <= 0 || a.B <= 0) return 0;
  LVSR_CHECK(a.ndir == 1 || a.ndir == 2, "bigru backward: %d directions (1 or 2)", a.ndir);
  const int rc = a.ndir == 1 ? launch_bwd_width<1>(a, stream) : launch_bwd_width<2>(a, stream);
  if (rc == 0 && cs_out) *cs_out = a.D / UC;   // the cluster size that ran
  return rc;
}

}  // namespace lvsr
