// Filterbank front end: Kaldi's compute-fbank-feats --use-energy | add-deltas | global CMVN, the features the recipes
// feed the recognizer (exp/wsj/write_hdf_dataset.sh:94-105).  The definition is restated in DESIGN §1 (j).
//
// Two passes:
//   fbank_frames_kernel: one CTA per (utterance row, run of kRun consecutive frames) stages the run's contiguous
//     sample span in shared memory with one bulk async copy, so overlapping frames read HBM once.  A warp per frame
//     dithers, removes the DC offset, takes the raw energy, pre-emphasises and windows the frame, runs a P-point real
//     FFT as a P/2-point complex radix-2 FFT plus the real split (twiddles tabulated in double on the host), sums
//     the power spectrum over each mel bin's nonzero range and takes the logs -> raw rows [T, B, D0].
//   fbank_finish_kernel: deltas with clamped frame indices, CMVN, the time-major features [T, B, D] and the mask;
//     frames past an utterance's end are written as exact zeros.
// The CMVN statistics are float64 partial sums per CTA over fixed row ranges, reduced in a fixed order.
#include <cfloat>
#include <algorithm>
#include <cmath>
#include <memory>
#include <vector>

#include <curand_kernel.h>

#include "common.cuh"
#include "lvsr_b200.h"

using namespace lvsr;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kRun = 16;                          // frames per CTA: two per warp
constexpr int kMaxP = LVSR_FBANK_MAX_PADDED;
constexpr int kCmvnCtas = 264;                    // partial sums of the CMVN accumulation (two per H100 SM)
constexpr int kMaxTaps = 32;                      // 2 * order * window + 1 <= 25 taps per delta order
constexpr int kMaxSmem = 226 * 1024;               // dynamic shared memory opt-in: 227 KB less the static barrier
constexpr unsigned kTagDither = 0xF8u << 24;      // stream tag of the dither draws (noise.cu tags its draws likewise)

struct DeltaScales { float s[LVSR_FBANK_MAX_DELTA_ORDER + 1][kMaxTaps]; };

struct MelBin { int first, count, woff; };

// N(0, 1) dither of samples 4g .. 4g+3 of frame t of utterance row b
__device__ __forceinline__ void dither4(unsigned long long seed, int b, int t, int g, float e[4]) {
  const uint4 ctr = make_uint4((unsigned)g, (unsigned)t, (unsigned)b, kTagDither);
  const uint4 r = curand_Philox4x32_10(ctr, make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
  const float2 a = box_muller(r.x, r.y), c = box_muller(r.z, r.w);
  e[0] = a.x; e[1] = a.y; e[2] = c.x; e[3] = c.y;
}

__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

struct FrameParams {
  const float* samples;       // [B, stride]
  long long stride;
  const int* frames;          // [B]
  float* raw;                 // [T, B, D0]
  const float* window;        // [W]
  const float2* twiddle;      // [P / 2]: exp(-2 pi i k / P)
  const MelBin* bins;         // [nbins]
  const float* weights;
  int B, W, S, P, log2n, nbins, D0;
  int use_energy, raw_energy, remove_dc, use_power;
  float dither, preemph, log_energy_floor;    // log_energy_floor: -inf when energy_floor is 0
  unsigned long long seed;
};

// shared memory of fbank_frames_kernel: per warp a frame buffer [kMaxP] floats and a complex buffer [kMaxP / 2]
// float2, the window (W rounded up to 4), the twiddles [P / 2] float2, then the sample span of the run (+ 4 for the
// alignment of its start)
static size_t frames_smem(int W, int S, int P) {
  return sizeof(float) * ((size_t)kWarps * 2 * kMaxP + ((W + 3) & ~3) + P + ((size_t)(kRun - 1) * S + W + 8));
}

__global__ void __launch_bounds__(kThreads) fbank_frames_kernel(const FrameParams p) {
  extern __shared__ __align__(16) float sm[];
  __shared__ __align__(8) unsigned long long bar;
  const int b = blockIdx.y, t0 = blockIdx.x * kRun;
  const int nf = p.frames[b];
  if (t0 >= nf) return;                           // padded frames: written by the finishing pass
  const int nrun = min(kRun, nf - t0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* fr = sm + warp * (2 * kMaxP);
  float2* z = reinterpret_cast<float2*>(fr + kMaxP);
  float* win = sm + kWarps * 2 * kMaxP;
  float2* tw = reinterpret_cast<float2*>(win + ((p.W + 3) & ~3));
  float* span = reinterpret_cast<float*>(tw + p.P / 2);

  // the run's samples [t0 S, (t0 + nrun - 1) S + W), widened to 16-byte boundaries (the row stride is a multiple of
  // 4 floats, so the widened span stays inside row b)
  const long long g0 = (long long)b * p.stride + (long long)t0 * p.S;
  const long long ga = g0 & ~3ll;
  const long long ge = ((long long)b * p.stride + (long long)(t0 + nrun - 1) * p.S + p.W + 3) & ~3ll;
  const uint32_t bytes = (uint32_t)((ge - ga) * sizeof(float));
  const uint32_t mb = smem_addr(&bar);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;\n" ::"r"(mb) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(mb), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                 ::"r"(smem_addr(span)), "l"(p.samples + ga), "r"(bytes), "r"(mb) : "memory");
  }
  for (int i = threadIdx.x; i < p.W; i += kThreads) win[i] = p.window[i];
  for (int i = threadIdx.x; i < p.P / 2; i += kThreads) tw[i] = p.twiddle[i];
  __syncthreads();                                // the barrier's init and the tables are visible to every thread
  for (uint32_t ok = 0, spins = 0; !ok;) {
    asm volatile("{\n\t.reg .pred q;\n\tmbarrier.try_wait.parity.shared::cta.b64 q, [%1], 0;\n\tselp.u32 %0, 1, 0, q;\n\t}\n"
                 : "=r"(ok) : "r"(mb) : "memory");
    if (!ok && ++spins > (1u << 24)) __trap();    // a lost transfer must fail the launch, not hang the GPU
  }

  const int N = p.P / 2;
  const int groups = (p.W + 3) >> 2;
  for (int l = warp; l < nrun; l += kWarps) {
    const int t = t0 + l;
    const float* src = span + (g0 - ga) + (long long)l * p.S;
    // 1. dither the frame's copy; 2. its mean
    float sum = 0.f;
    for (int g = lane; g < groups; g += 32) {
      float e[4] = {0.f, 0.f, 0.f, 0.f};
      if (p.dither != 0.f) dither4(p.seed, b, t, g, e);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = 4 * g + q;
        if (i < p.W) {
          const float v = fmaf(p.dither, e[q], src[i]);
          fr[i] = v;
          sum += v;
        }
      }
    }
    const float mean = p.remove_dc ? warp_sum(sum) / (float)p.W : 0.f;
    __syncwarp();
    // 3. raw energy; 4. pre-emphasis (x[i] - p x[i-1] of the DC-free frame, x[0] - p x[0]); 5. window; 6. windowed
    // energy; the frame goes into the complex buffer as z[n] = x[2n] + i x[2n+1], at the bit-reversed index of n
    float e_raw = 0.f, e_win = 0.f;
    for (int i = lane; i < p.P; i += 32) {
      float w = 0.f;
      if (i < p.W) {
        const float x = fr[i] - mean;
        const float xp = i > 0 ? fr[i - 1] - mean : x;
        e_raw = fmaf(x, x, e_raw);
        w = fmaf(-p.preemph, xp, x) * win[i];
        e_win = fmaf(w, w, e_win);
      }
      const int n = __brev((unsigned)(i >> 1)) >> (32 - p.log2n);
      reinterpret_cast<float*>(z + n)[i & 1] = w;
    }
    const float energy = warp_sum(p.raw_energy ? e_raw : e_win);
    __syncwarp();
    // 7. N-point complex FFT, decimation in time
    for (int s = 0, h = 1; s < p.log2n; ++s, h <<= 1) {
      for (int k = lane; k < N / 2; k += 32) {
        const int j = k & (h - 1);
        const int i0 = ((k >> s) << (s + 1)) + j, i1 = i0 + h;
        const float2 w = tw[j * (N >> s)];
        const float2 a = z[i0], c = z[i1];
        const float2 cw = make_float2(c.x * w.x - c.y * w.y, c.x * w.y + c.y * w.x);
        z[i0] = make_float2(a.x + cw.x, a.y + cw.y);
        z[i1] = make_float2(a.x - cw.x, a.y - cw.y);
      }
      __syncwarp();
    }
    // real split: X_k = E_k + e^{-2 pi i k / P} O_k, E = (Z_k + conj Z_{N-k}) / 2, O = -i (Z_k - conj Z_{N-k}) / 2;
    // the power spectrum of bins 0 .. N-1 (the Nyquist bin is never used) overwrites the frame buffer
    for (int k = lane; k < N; k += 32) {
      float re, im;
      if (k == 0) {
        re = z[0].x + z[0].y;
        im = 0.f;
      } else {
        const float2 a = z[k], c = z[N - k];
        const float er = 0.5f * (a.x + c.x), ei = 0.5f * (a.y - c.y);
        const float orr = 0.5f * (a.y + c.y), oi = -0.5f * (a.x - c.x);
        const float2 w = tw[k];
        re = er + (w.x * orr - w.y * oi);
        im = ei + (w.x * oi + w.y * orr);
      }
      const float pw = fmaf(re, re, im * im);
      fr[k] = p.use_power ? pw : sqrtf(pw);
    }
    __syncwarp();
    // mel banks over each bin's nonzero range, then the logs
    float* row = p.raw + ((size_t)t * p.B + b) * p.D0;
    for (int m = lane; m < p.nbins; m += 32) {
      const MelBin mbin = p.bins[m];
      float acc = 0.f;
      for (int i = 0; i < mbin.count; ++i) acc = fmaf(__ldg(p.weights + mbin.woff + i), fr[mbin.first + i], acc);
      row[p.use_energy + m] = logf(fmaxf(acc, FLT_EPSILON));
    }
    if (p.use_energy && lane == 0) {
      row[0] = fmaxf(logf(fmaxf(energy, FLT_EPSILON)), p.log_energy_floor);
    }
    __syncwarp();                                 // fr and z are rewritten by the warp's next frame
  }
}

// scale and offset of column c: x' = x scale + offset, computed in float64 from the stats (Kaldi's ApplyCmvn)
__device__ __forceinline__ void cmvn_coeffs(const double* stats, int D, float* sc, float* of) {
  const double n = stats[D];
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    const double mean = stats[c] / n;
    const double var = fmax(stats[D + 1 + c] / n - mean * mean, 1e-20);
    const double scale = 1.0 / sqrt(var);
    sc[c] = (float)scale;
    of[c] = (float)(-mean * scale);
  }
  __syncthreads();
}

// deltas, CMVN and the write of features [T, B, D] and mask [T, B]
__global__ void __launch_bounds__(kThreads) fbank_finish_kernel(const float* __restrict__ raw, const int* __restrict__ frames,
                                                                 float* __restrict__ out, float* __restrict__ mask,
                                                                 const double* __restrict__ stats, int T, int B, int D0,
                                                                 int order, int window, const DeltaScales scales) {
  extern __shared__ float coef[];                 // [2 D] when stats
  const int D = D0 * (order + 1);
  if (stats) cmvn_coeffs(stats, D, coef, coef + D);
  const long long n = (long long)T * B * D;
  for (long long e = blockIdx.x * (long long)kThreads + threadIdx.x; e < n; e += (long long)gridDim.x * kThreads) {
    const long long r = e / D;
    const int c = (int)(e - r * D);
    const int t = (int)(r / B), b = (int)(r - (long long)t * B);
    const int nf = frames[b];
    float v = 0.f;
    if (t < nf) {
      const int o = c / D0, j = c - o * D0;
      if (o == 0) {
        v = raw[r * D0 + j];
      } else {
        const int reach = o * window;
        for (int k = -reach; k <= reach; ++k) {
          const int tt = min(max(t + k, 0), nf - 1);
          v = fmaf(scales.s[o][k + reach], raw[((size_t)tt * B + b) * D0 + j], v);
        }
      }
      if (stats) v = fmaf(v, coef[c], coef[D + c]);
    }
    out[e] = v;
    if (c == 0) mask[r] = t < nf ? 1.f : 0.f;
  }
}

// per CTA: float64 sums of x and x^2 of the masked-in rows of its fixed range, and their count -> part[cta][2][D + 1]
__global__ void __launch_bounds__(kThreads) cmvn_partial_kernel(const float* __restrict__ x, const float* __restrict__ mask,
                                                                long long rows, int D, double* __restrict__ part) {
  const long long chunk = (rows + gridDim.x - 1) / gridDim.x;
  const long long r0 = blockIdx.x * chunk, r1 = min(rows, r0 + chunk);
  double* out = part + (size_t)blockIdx.x * 2 * (D + 1);
  for (int c = threadIdx.x; c <= D; c += kThreads) {
    double s0 = 0.0, s1 = 0.0;
    for (long long r = r0; r < r1; ++r) {
      if (mask && !(mask[r] > 0.5f)) continue;
      if (c == D) {
        s0 += 1.0;
      } else {
        const double v = x[r * D + c];
        s0 += v;
        s1 = fma(v, v, s1);
      }
    }
    out[c] = s0;
    out[D + 1 + c] = s1;
  }
}

// stats += the partial sums, added in CTA order
__global__ void __launch_bounds__(kThreads) cmvn_reduce_kernel(const double* __restrict__ part, int nparts, int D,
                                                               double* __restrict__ stats) {
  for (int c = threadIdx.x; c < 2 * (D + 1); c += kThreads) {
    double s = 0.0;
    for (int i = 0; i < nparts; ++i) s += part[(size_t)i * 2 * (D + 1) + c];
    stats[c] += s;
  }
}

__global__ void __launch_bounds__(kThreads) cmvn_apply_kernel(float* __restrict__ x, const float* __restrict__ mask,
                                                              long long rows, int D, const double* __restrict__ stats) {
  extern __shared__ float coef[];
  cmvn_coeffs(stats, D, coef, coef + D);
  const long long n = rows * D;
  for (long long e = blockIdx.x * (long long)kThreads + threadIdx.x; e < n; e += (long long)gridDim.x * kThreads) {
    const long long r = e / D;
    const int c = (int)(e - r * D);
    if (!mask || mask[r] > 0.5f) x[e] = fmaf(x[e], coef[c], coef[D + c]);
  }
}

__global__ void __launch_bounds__(kThreads) dither_sample_kernel(float* __restrict__ out, int B, int T, int W,
                                                                 unsigned long long seed) {
  const int groups = (W + 3) >> 2;
  const long long n = (long long)B * T * groups;
  for (long long e = blockIdx.x * (long long)kThreads + threadIdx.x; e < n; e += (long long)gridDim.x * kThreads) {
    const int g = (int)(e % groups);
    const long long bt = e / groups;
    const int t = (int)(bt % T), b = (int)(bt / T);
    float d[4];
    dither4(seed, b, t, g, d);
    for (int q = 0; q < 4 && 4 * g + q < W; ++q) out[bt * W + 4 * g + q] = d[q];
  }
}

double mel_scale(double f) { return 1127.0 * std::log(1.0 + f / 700.0); }

int elementwise_grid(long long n) {
  const long long want = (n + kThreads - 1) / kThreads;
  return (int)std::max(1ll, std::min(want, (long long)device_sm_count() * 8));
}

}  // namespace

struct lvsr_frontend {
  lvsr_fbank_options opt;
  int device = 0;
  cudaStream_t stream = nullptr;
  int W = 0, S = 0, P = 0, log2n = 0, D0 = 0, D = 0;
  DeltaScales scales = {};
  DeviceBuffer<float> table;        // window [W] | twiddles [P / 2] float2 | mel weights
  DeviceBuffer<MelBin> bins;
  const float2* twiddle = nullptr;
  const float* weights = nullptr;
  DeviceBuffer<double> part;        // [kCmvnCtas][2][D + 1]
  DeviceBuffer<float> raw;          // [T, B, D0], grown on demand
  DeviceBuffer<int> frames;         // [B], grown on demand
};

extern "C" {

int lvsr_frontend_create(const lvsr_fbank_options* o, lvsr_frontend** out) {
  LVSR_CHECK(o && out, "frontend_create: null argument");
  *out = nullptr;
  LVSR_CHECK(o->snip_edges == 1, "snip_edges false is not supported (only snip_edges true)");
  LVSR_CHECK(o->vtln_warp == 1.0, "VTLN warping is not supported (vtln_warp must be 1, got %g)", o->vtln_warp);
  LVSR_CHECK(o->htk_compat == 0, "htk_compat true is not supported");
  LVSR_CHECK(o->use_log_fbank == 1, "use_log_fbank false is not supported (only log filterbanks)");
  LVSR_CHECK(std::isfinite(o->sample_frequency) && o->sample_frequency > 0, "sample_frequency must be > 0");
  LVSR_CHECK(o->frame_length > 0 && o->frame_shift > 0, "frame_length and frame_shift must be > 0");
  const double fs = o->sample_frequency;
  const long long W = (long long)(fs * 0.001 * o->frame_length), S = (long long)(fs * 0.001 * o->frame_shift);
  LVSR_CHECK(W >= 2 && S >= 1, "frame_length %g ms / frame_shift %g ms give %lld / %lld samples", o->frame_length,
             o->frame_shift, W, S);
  long long P = 1;
  while (P < W) P <<= 1;
  LVSR_CHECK(P <= kMaxP, "frame_length %g ms is %lld samples: longer than the %d-point FFT supports", o->frame_length, W,
             kMaxP);
  LVSR_CHECK(o->round_to_power_of_two == 1 || P == W,
             "round_to_power_of_two false needs a frame of a power-of-two length (got %lld samples)", W);
  LVSR_CHECK(P >= 4, "frame of %lld samples too short", W);
  LVSR_CHECK(frames_smem((int)W, (int)S, (int)P) <= (size_t)kMaxSmem,
             "frame_shift %g ms (%lld samples) is too long for a run of %d frames in shared memory", o->frame_shift, S,
             kRun);
  LVSR_CHECK(o->dither >= 0 && std::isfinite(o->dither), "dither must be >= 0");
  LVSR_CHECK(o->preemphasis_coefficient >= 0 && o->preemphasis_coefficient <= 1, "preemphasis_coefficient must be in [0, 1]");
  LVSR_CHECK(o->window_type >= LVSR_WINDOW_POVEY && o->window_type <= LVSR_WINDOW_RECTANGULAR,
             "window_type %d unsupported (povey, hamming, hanning or rectangular)", o->window_type);
  LVSR_CHECK(o->energy_floor >= 0, "energy_floor must be >= 0");
  LVSR_CHECK(o->num_mel_bins >= 3, "num_mel_bins must be at least 3");
  LVSR_CHECK(o->delta_order >= 0 && o->delta_order <= LVSR_FBANK_MAX_DELTA_ORDER, "delta_order %d not in [0, %d]",
             o->delta_order, (int)LVSR_FBANK_MAX_DELTA_ORDER);
  LVSR_CHECK(o->delta_order == 0 || (o->delta_window >= 1 && o->delta_window <= LVSR_FBANK_MAX_DELTA_WINDOW),
             "delta_window %d not in [1, %d]", o->delta_window, (int)LVSR_FBANK_MAX_DELTA_WINDOW);
  for (int32_t flag : {o->remove_dc_offset, o->use_energy, o->raw_energy, o->use_power})
    LVSR_CHECK(flag == 0 || flag == 1, "remove_dc_offset, use_energy, raw_energy and use_power must be 0 or 1");
  const double nyq = 0.5 * fs;
  const double lo = o->low_freq, hi = o->high_freq > 0 ? o->high_freq : nyq + o->high_freq;
  LVSR_CHECK(lo >= 0 && lo < nyq && hi > 0 && hi <= nyq && hi > lo,
             "bad mel band edges: low_freq %g, high_freq %g (effective %g) at sample_frequency %g", lo, o->high_freq, hi, fs);
  // mel banks: bins 0 .. P/2 - 1 at i fs / P, triangles in mel between num_mel_bins + 1 equal steps
  const int N = (int)(P / 2), nb = o->num_mel_bins;
  const double mlo = mel_scale(lo), delta = (mel_scale(hi) - mlo) / (nb + 1);
  std::vector<MelBin> bins(nb);
  std::vector<float> weights;
  for (int m = 0; m < nb; ++m) {
    const double left = mlo + m * delta, centre = left + delta, right = centre + delta;
    bins[m] = MelBin{-1, 0, (int)weights.size()};
    for (int i = 0; i < N; ++i) {
      const double mel = mel_scale(i * fs / (double)P);
      if (mel > left && mel < right) {
        if (bins[m].first < 0) bins[m].first = i;
        weights.push_back((float)(mel <= centre ? (mel - left) / (centre - left) : (right - mel) / (right - centre)));
        bins[m].count = i - bins[m].first + 1;
      }
    }
    LVSR_CHECK(bins[m].count > 0, "num_mel_bins %d too large: mel bin %d has no FFT bin", nb, m);
  }
  int dev_count = 0;
  LVSR_CUDA_OK(cudaGetDeviceCount(&dev_count));
  LVSR_CHECK(dev_count > 0, "no CUDA device: the front end has no CPU fallback");

  std::unique_ptr<lvsr_frontend> f(new lvsr_frontend());   // deleted with its buffers on a failed return
  f->opt = *o;
  f->W = (int)W;
  f->S = (int)S;
  f->P = (int)P;
  while ((1 << f->log2n) < N) ++f->log2n;
  f->D0 = nb + (o->use_energy ? 1 : 0);
  f->D = f->D0 * (o->delta_order + 1);
  // add-deltas: scales_0 = [1], scales_i = conv(scales_{i-1}, [-w .. w]) / sum_{j=-w..w} j^2
  {
    std::vector<double> prev{1.0};
    const int w = o->delta_window;
    double norm = 0.0;
    for (int j = -w; j <= w; ++j) norm += (double)j * j;
    f->scales.s[0][0] = 1.f;
    for (int ord = 1; ord <= o->delta_order; ++ord) {
      std::vector<double> cur(prev.size() + 2 * w, 0.0);
      for (size_t a = 0; a < prev.size(); ++a)
        for (int j = -w; j <= w; ++j) cur[a + j + w] += prev[a] * j / norm;
      for (size_t a = 0; a < cur.size(); ++a) f->scales.s[ord][a] = (float)cur[a];
      prev.swap(cur);
    }
  }
  // window, twiddles and mel weights in one table, laid out as fbank_frames_kernel reads them
  std::vector<float> table;
  const double a = 2.0 * M_PI / (double)(W - 1);
  for (int i = 0; i < W; ++i) {
    double v = 1.0;
    switch (o->window_type) {
      case LVSR_WINDOW_POVEY: v = std::pow(0.5 - 0.5 * std::cos(a * i), 0.85); break;
      case LVSR_WINDOW_HAMMING: v = 0.54 - 0.46 * std::cos(a * i); break;
      case LVSR_WINDOW_HANNING: v = 0.5 - 0.5 * std::cos(a * i); break;
      default: break;
    }
    table.push_back((float)v);
  }
  while (table.size() % 2) table.push_back(0.f);
  const size_t tw_off = table.size();
  for (int k = 0; k < N; ++k) {
    table.push_back((float)std::cos(2.0 * M_PI * k / (double)P));
    table.push_back((float)-std::sin(2.0 * M_PI * k / (double)P));
  }
  const size_t w_off = table.size();
  table.insert(table.end(), weights.begin(), weights.end());
  cudaError_t e = cudaGetDevice(&f->device);
  if (e == cudaSuccess) e = f->table.alloc(table.size() * sizeof(float));
  if (e == cudaSuccess) e = f->bins.alloc(nb * sizeof(MelBin));
  if (e == cudaSuccess) e = f->part.alloc((size_t)kCmvnCtas * 2 * (f->D + 1) * sizeof(double));
  if (e == cudaSuccess) e = cudaMemcpy(f->table.get(), table.data(), table.size() * sizeof(float), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(f->bins.get(), bins.data(), nb * sizeof(MelBin), cudaMemcpyHostToDevice);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(fbank_frames_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
  if (e != cudaSuccess) return set_error("frontend_create: %s", cudaGetErrorString(e));
  f->twiddle = reinterpret_cast<const float2*>(f->table.get() + tw_off);
  f->weights = f->table.get() + w_off;
  *out = f.release();
  return 0;
}

int lvsr_frontend_destroy(lvsr_frontend* f) {
  if (!f) return 0;
  DeviceGuard guard(f);
  cudaStreamSynchronize(f->stream);
  delete f;
  return 0;
}

int64_t lvsr_frontend_num_frames(const lvsr_frontend* f, int64_t num_samples) {
  if (!f) return -1;
  return num_samples < f->W ? 0 : 1 + (num_samples - f->W) / f->S;
}

int lvsr_frontend_feature_dim(const lvsr_frontend* f) { return f ? f->D : -1; }

int lvsr_frontend_compute(lvsr_frontend* f, const float* samples_dev, int64_t row_stride, const int64_t* lengths_host,
                          int32_t B, int32_t T, float* features_dev, float* mask_dev, const double* cmvn_stats_dev,
                          void* stream) {
  LVSR_CHECK(f && samples_dev && lengths_host && features_dev && mask_dev, "frontend_compute: null argument");
  LVSR_CHECK(B >= 1 && T >= 1, "frontend_compute: B %d and T %d must be >= 1", B, T);
  LVSR_CHECK(row_stride >= 4 && row_stride % 4 == 0 && ((uintptr_t)samples_dev & 15) == 0,
             "frontend_compute: samples must be 16-byte aligned with a row stride that is a multiple of 4 (got %lld)",
             (long long)row_stride);
  std::vector<int> frames(B);
  for (int b = 0; b < B; ++b) {
    LVSR_CHECK(lengths_host[b] <= row_stride, "utterance %d: %lld samples exceed the row stride %lld", b,
               (long long)lengths_host[b], (long long)row_stride);
    const int64_t nf = lvsr_frontend_num_frames(f, lengths_host[b]);
    LVSR_CHECK(nf >= 1, "utterance %d is shorter than one frame (%lld samples, a frame is %d)", b,
               (long long)lengths_host[b], f->W);
    LVSR_CHECK(nf <= T, "utterance %d has %lld frames, more than T = %d", b, (long long)nf, T);
    frames[b] = (int)nf;
  }
  DeviceGuard guard(f);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_stream(f, st)) return rc;
  LVSR_CUDA_OK(f->frames.grow((size_t)B * sizeof(int), f->stream));
  LVSR_CUDA_OK(f->raw.grow((size_t)T * B * f->D0 * sizeof(float), f->stream));
  LVSR_CUDA_OK(cudaMemcpyAsync(f->frames.get(), frames.data(), B * sizeof(int), cudaMemcpyHostToDevice, st));
  ProfScope prof("fbank", st);
  FrameParams p;
  p.samples = samples_dev;
  p.stride = row_stride;
  p.frames = f->frames.get();
  p.raw = f->raw.get();
  p.window = f->table.get();
  p.twiddle = f->twiddle;
  p.bins = f->bins.get();
  p.weights = f->weights;
  p.B = B;
  p.W = f->W;
  p.S = f->S;
  p.P = f->P;
  p.log2n = f->log2n;
  p.nbins = f->opt.num_mel_bins;
  p.D0 = f->D0;
  p.use_energy = f->opt.use_energy;
  p.raw_energy = f->opt.raw_energy;
  p.remove_dc = f->opt.remove_dc_offset;
  p.use_power = f->opt.use_power;
  p.dither = (float)f->opt.dither;
  p.preemph = (float)f->opt.preemphasis_coefficient;
  p.log_energy_floor = f->opt.energy_floor > 0 ? (float)std::log(f->opt.energy_floor) : -INFINITY;
  p.seed = f->opt.seed;
  const dim3 grid((unsigned)ceil_div(T, kRun), (unsigned)B);
  fbank_frames_kernel<<<grid, kThreads, frames_smem(f->W, f->S, f->P), st>>>(p);
  LVSR_LAUNCH_CHECK();
  const long long n = (long long)T * B * f->D;
  fbank_finish_kernel<<<elementwise_grid(n), kThreads, cmvn_stats_dev ? 2 * f->D * sizeof(float) : 0, st>>>(
      f->raw.get(), f->frames.get(), features_dev, mask_dev, cmvn_stats_dev, T, B, f->D0, f->opt.delta_order, f->opt.delta_window,
      f->scales);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int lvsr_frontend_accumulate_cmvn(lvsr_frontend* f, const float* features_dev, const float* mask_dev, int32_t T,
                                  int32_t B, double* stats_dev, void* stream) {
  LVSR_CHECK(f && features_dev && stats_dev && T >= 1 && B >= 1, "frontend_accumulate_cmvn: bad arguments");
  DeviceGuard guard(f);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_stream(f, st)) return rc;
  const long long rows = (long long)T * B;
  const int nparts = (int)std::min<long long>(kCmvnCtas, rows);
  cmvn_partial_kernel<<<nparts, kThreads, 0, st>>>(features_dev, mask_dev, rows, f->D, f->part.get());
  LVSR_LAUNCH_CHECK();
  cmvn_reduce_kernel<<<1, kThreads, 0, st>>>(f->part.get(), nparts, f->D, stats_dev);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int lvsr_frontend_apply_cmvn(lvsr_frontend* f, float* features_dev, const float* mask_dev, int32_t T, int32_t B,
                             const double* stats_dev, void* stream) {
  LVSR_CHECK(f && features_dev && stats_dev && T >= 1 && B >= 1, "frontend_apply_cmvn: bad arguments");
  DeviceGuard guard(f);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_stream(f, st)) return rc;
  const long long rows = (long long)T * B;
  cmvn_apply_kernel<<<elementwise_grid(rows * f->D), kThreads, 2 * f->D * sizeof(float), st>>>(features_dev, mask_dev,
                                                                                             rows, f->D, stats_dev);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int lvsr_frontend_dither_sample(lvsr_frontend* f, int32_t B, int32_t T, float* draws_dev, void* stream) {
  LVSR_CHECK(f && draws_dev && B >= 1 && T >= 1, "frontend_dither_sample: bad arguments");
  DeviceGuard guard(f);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_stream(f, st)) return rc;
  const long long n = (long long)B * T * ((f->W + 3) >> 2);
  dither_sample_kernel<<<elementwise_grid(n), kThreads, 0, st>>>(draws_dev, B, T, f->W, f->opt.seed);
  LVSR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
