// Alignment statistics of the validation pass: weights_entropy and weights_penalty (lvsr/expressions.py:4-25 as
// lvsr/main.py:385-388 monitors them), summed over a batch of teacher-forced alignments [L, B, T'].
//
// One launch.  CTA b scans row b step by step: each thread owns a contiguous run of positions, the cumulative sum over
// t is a block scan, and the cumsum of step i - 1 stays in shared memory (at the positions the same thread owns) while
// step i is scanned, so the weights are read once.  Every sum is float64 in a fixed order; the CTA that finishes last
// adds the rows' partial sums in row order, so the result does not depend on scheduling.
#include <algorithm>

#include "model.h"

using namespace lvsr;

namespace {

constexpr int AS_THREADS = 256;

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// part [2 B]: per row (entropy, penalty); done: CTAs finished (the last one resets it); out [2]
__global__ void __launch_bounds__(AS_THREADS) alignment_stats_kernel(const float* __restrict__ w, const float* mask, int L,
                                                                     int B, int Tp, double* part, unsigned* done,
                                                                     double* out) {
  extern __shared__ double prev[];                 // [Tp] cumsum of step i - 1
  __shared__ double wsum[AS_THREADS / 32];
  __shared__ double red[2][AS_THREADS / 32];
  __shared__ bool last;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int chunk = (Tp + AS_THREADS - 1) / AS_THREADS;
  const int t0 = min(Tp, tid * chunk), t1 = min(Tp, t0 + chunk);
  double ent = 0.0, pen = 0.0;
  for (int i = 0; i < L; ++i) {
    const float* row = w + ((long long)i * B + b) * Tp;
    const double mk = mask ? (double)mask[(long long)i * B + b] : 1.0;
    double s = 0.0, e = 0.0;
    for (int t = t0; t < t1; ++t) {
      const double v = row[t];
      s += v;
      e += v * log(v + 1e-7);
    }
    // exclusive prefix of s over the threads: warp scan, then the sums of the warps before this one
    double incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    double c = incl - s;
    for (int q = 0; q < warp; ++q) c += wsum[q];
    double p = 0.0;
    for (int t = t0; t < t1; ++t) {
      c += row[t];
      if (i > 0) p += fmax(c - prev[t], 0.0);
      prev[t] = c;
    }
    ent += mk * e;
    if (i > 0) pen += mk * p;
    __syncthreads();                               // wsum is rewritten by the next step
  }
  ent = warp_sum_f64(ent);
  pen = warp_sum_f64(pen);
  if (lane == 0) { red[0][warp] = ent; red[1][warp] = pen; }
  __syncthreads();
  if (tid == 0) {
    double se = 0.0, sp = 0.0;
    for (int q = 0; q < AS_THREADS / 32; ++q) { se += red[0][q]; sp += red[1][q]; }
    part[2 * b] = se;
    part[2 * b + 1] = sp;
    __threadfence();                               // the partials are visible before the count says so
    last = atomicAdd(done, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (last && tid == 0) {
    double se = 0.0, sp = 0.0;
    for (int r = 0; r < B; ++r) { se += __ldcg(part + 2 * r); sp += __ldcg(part + 2 * r + 1); }
    out[0] = se;
    out[1] = sp;
    *done = 0;
  }
}

}  // namespace

extern "C" int lvsr_alignment_stats(lvsr_model* m, const float* weights_dev, const float* labels_mask_dev, int32_t L,
                                    int32_t B, int32_t Tp, double* out_dev, void* stream) {
  DeviceGuard device_guard(m);
  LVSR_CHECK(m && weights_dev && out_dev && L > 0 && B > 0 && Tp > 0, "alignment_stats: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_stream(m, st)) return rc;
  const size_t smem = (size_t)Tp * sizeof(double);
  int dev = 0, smem_max = 0;
  LVSR_CUDA_OK(cudaGetDevice(&dev));
  LVSR_CUDA_OK(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  LVSR_CHECK(smem + 1024 <= (size_t)smem_max, "alignment_stats: T' = %d exceeds the %d positions a CTA holds", Tp,
             (int)((smem_max - 1024) / sizeof(double)));
  const size_t need = 256 + 2 * (size_t)B * sizeof(double);
  if (need > m->align_mem.bytes()) {              // regrown: the previous call may still use the partials
    LVSR_CUDA_OK(m->align_mem.grow(need, st));    // a failed allocation leaves it empty: the next call regrows it
    const cudaError_t e = cudaMemsetAsync(m->align_mem.get(), 0, 256, st);
    if (e != cudaSuccess) {
      m->align_mem.reset();                       // so does a counter that was not zeroed
      return set_error("cudaMemsetAsync(alignment_stats counter) failed: %s", cudaGetErrorString(e));
    }
  }
  if (smem > 48 * 1024)
    LVSR_CUDA_OK(cudaFuncSetAttribute(alignment_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  unsigned* done = static_cast<unsigned*>(m->align_mem.get());
  double* part = reinterpret_cast<double*>(static_cast<char*>(m->align_mem.get()) + 256);
  alignment_stats_kernel<<<B, AS_THREADS, smem, st>>>(weights_dev, labels_mask_dev, L, B, Tp, part, done, out_dev);
  LVSR_LAUNCH_CHECK();
  return 0;
}
