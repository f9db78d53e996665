// Adaptive weight noise (Graves 2011, "Practical Variational Inference for Neural Networks"): apply_adaptive_noise of
// lvsr/graph.py:71-251 as lvsr/main.py:425-460 applies it to every parameter of the recognizer.
//
// Per parameter p (every entry of the flat layout, padding excluded) a log-variance ls2 of the same shape
// (graph.py:173-179), S = 2048 (log_sigma_scale, :159):
//   s2 = exp(S ls2),  p_noisy = p + eps sqrt(s2), eps ~ N(0, 1) fresh every update                      :178-183
//   prior_u = sum(p) / n,  prior_s2 = (sum(s2) + sum((p - prior_u)^2)) / n   over ALL parameters      :186-198
//   LC = coef / N sum[0.5 (log prior_s2 - S ls2) + ((p - prior_u)^2 + s2 - prior_s2) / (2 prior_s2)]   :206-214
//   grad p   = coef (p - prior_u) / (N prior_s2) + g                                                   :240-241
//   grad ls2 = coef 0.5 S / N (s2 / prior_s2 - 1) + 0.5 S s2 g^2                                       :243-247
// with g the task gradient at p_noisy, the priors constants of the gradients, and g^2 the reference's "diagonal
// Hessian" (not the reparameterisation gradient eps g).  The reference draws eps from Theano's MRG31k3p streams;
// here it is Philox-4x32-10 keyed by (seed, update counter, flat index), Box-Muller in fp32, so that every
// data-parallel rank draws the same noise without communication.
//
// The sample pass (one read of p and ls2, one write of p_noisy) also accumulates float64 partial sums of p, p^2, s2
// and ls2 per CTA; one CTA then reduces them in a fixed order, so priors and model cost are deterministic.
#include <curand_kernel.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "model.h"

using namespace lvsr;

namespace {

constexpr double kLogSigmaScale = 2048.0;      // graph.py:159
constexpr int kThreads = 256;
constexpr int kCtasPerParam = 32;              // grid (kCtasPerParam, parameters); the partial sums follow this grid

struct Span { long long offset, count; };

// Stream tags of the draws, in the high byte of the fourth Philox counter word (adaptive noise: 0, so its draws are
// those of an update counter below 2^24 * 2^32)
constexpr unsigned kTagDropout = 0xD0u << 24, kTagWeightNoise = 0x57u << 24;

// eps of the four flat elements 4q .. 4q+3 (a parameter starts at a multiple of 64, so a group never straddles two)
__device__ __forceinline__ void eps4(unsigned long long seed, unsigned long long update, unsigned long long q, float e[4],
                                     unsigned tag = 0) {
  const uint4 ctr = make_uint4((unsigned)q, (unsigned)(q >> 32), (unsigned)update, (unsigned)(update >> 32) ^ tag);
  const uint4 r = curand_Philox4x32_10(ctr, make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
  const float2 a = box_muller(r.x, r.y), b = box_muller(r.z, r.w);
  e[0] = a.x; e[1] = a.y; e[2] = b.x; e[3] = b.y;
}

__device__ __forceinline__ double block_sum(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < kThreads / 32; ++w) s += red[w];
  return s;
}

// p_noisy = p + eps exp(1024 ls2) (= eps sqrt(s2)); per CTA the sums of p, p^2, s2, ls2 -> part[4 * cta + k]
__global__ void __launch_bounds__(kThreads) noise_sample_kernel(const float* __restrict__ mean, const float* __restrict__ ls2,
                                                                float* __restrict__ noisy, const Span* spans,
                                                                unsigned long long seed, unsigned long long update,
                                                                double* part) {
  __shared__ double red[kThreads / 32];
  const Span sp = spans[blockIdx.y];
  double sp1 = 0.0, sp2 = 0.0, ss2 = 0.0, sl = 0.0;
  const long long groups = (sp.count + 3) >> 2;
  for (long long gq = blockIdx.x * (long long)kThreads + threadIdx.x; gq < groups; gq += (long long)gridDim.x * kThreads) {
    const long long i0 = sp.offset + 4 * gq;
    const float4 p4 = *reinterpret_cast<const float4*>(mean + i0);
    const float4 l4 = *reinterpret_cast<const float4*>(ls2 + i0);
    const float p[4] = {p4.x, p4.y, p4.z, p4.w}, l[4] = {l4.x, l4.y, l4.z, l4.w};
    float e[4], o[4];
    eps4(seed, update, (unsigned long long)i0 >> 2, e);
    const long long valid = sp.count - 4 * gq;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      o[j] = 0.f;                                   // the padding after a parameter stays zero
      if (j < valid) {
        const float sigma = expf(1024.f * l[j]);
        o[j] = fmaf(sigma, e[j], p[j]);
        sp1 += p[j];
        sp2 += (double)p[j] * p[j];
        ss2 += (double)sigma * sigma;
        sl += l[j];
      }
    }
    *reinterpret_cast<float4*>(noisy + i0) = make_float4(o[0], o[1], o[2], o[3]);
  }
  const double t0 = block_sum(sp1, red), t1 = block_sum(sp2, red), t2 = block_sum(ss2, red), t3 = block_sum(sl, red);
  if (threadIdx.x == 0) {
    double* out = part + 4 * ((size_t)blockIdx.y * gridDim.x + blockIdx.x);
    out[0] = t0; out[1] = t1; out[2] = t2; out[3] = t3;
  }
}

// fixed-order reduction of the partial sums -> stats [model cost, prior mean, prior variance, n]
__global__ void __launch_bounds__(kThreads) noise_prior_kernel(const double* part, int nparts, double n, double coef_over_n,
                                                               double* stats) {
  __shared__ double red[kThreads / 32];
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  for (int i = threadIdx.x; i < nparts; i += kThreads)
    for (int k = 0; k < 4; ++k) s[k] += part[4 * (size_t)i + k];
  double t[4];
  for (int k = 0; k < 4; ++k) t[k] = block_sum(s[k], red);
  if (threadIdx.x == 0) {
    const double u = t[0] / n;
    const double dev2 = t[1] - 2.0 * u * t[0] + n * u * u;      // sum (p - prior_u)^2
    const double ps2 = (t[2] + dev2) / n;
    stats[LVSR_NOISE_MODEL_COST] = coef_over_n * (0.5 * (n * log(ps2) - kLogSigmaScale * t[3]) + (dev2 + t[2] - n * ps2) / (2.0 * ps2));
    stats[LVSR_NOISE_PRIOR_MEAN] = u;
    stats[LVSR_NOISE_PRIOR_VARIANCE] = ps2;
    stats[3] = n;
  }
}

// both gradient groups from g = gscale * grads (the mean gradient at the noisy parameters); per CTA the sum of squares
// of the two into norm_part (null: not needed)
__global__ void __launch_bounds__(kThreads) noise_grad_kernel(float* __restrict__ grads, float* __restrict__ gls2,
                                                              const float* __restrict__ mean, const float* __restrict__ ls2,
                                                              const Span* spans, const double* stats, float gscale,
                                                              float coef_over_n, float* norm_part) {
  __shared__ double red[kThreads / 32];
  const Span sp = spans[blockIdx.y];
  const float u = (float)stats[LVSR_NOISE_PRIOR_MEAN];
  const float ps2 = (float)stats[LVSR_NOISE_PRIOR_VARIANCE];
  const float a = coef_over_n / ps2;
  const float half_s = 0.5f * (float)kLogSigmaScale;
  float sq = 0.f;
  for (long long i = blockIdx.x * (long long)kThreads + threadIdx.x; i < sp.count; i += (long long)gridDim.x * kThreads) {
    const long long o = sp.offset + i;
    const float g = grads[o] * gscale;
    const float s2 = expf((float)kLogSigmaScale * ls2[o]);
    const float gp = fmaf(a, mean[o] - u, g);
    const float gl = coef_over_n * half_s * (s2 / ps2 - 1.f) + half_s * s2 * g * g;
    grads[o] = gp;
    gls2[o] = gl;
    sq = fmaf(gp, gp, fmaf(gl, gl, sq));
  }
  if (!norm_part) return;
  const double t = block_sum(sq, red);
  if (threadIdx.x == 0) norm_part[(size_t)blockIdx.y * gridDim.x + blockIdx.x] = (float)t;
}

__global__ void __launch_bounds__(kThreads) noise_eps_kernel(float* __restrict__ eps, const Span* spans, unsigned long long seed,
                                                             unsigned long long update) {
  const Span sp = spans[blockIdx.y];
  const long long groups = (sp.count + 3) >> 2;
  for (long long gq = blockIdx.x * (long long)kThreads + threadIdx.x; gq < groups; gq += (long long)gridDim.x * kThreads) {
    const long long i0 = sp.offset + 4 * gq;
    float e[4];
    eps4(seed, update, (unsigned long long)i0 >> 2, e);
    for (int j = 0; j < 4 && 4 * gq + j < sp.count; ++j) eps[i0 + j] = e[j];
  }
}

__global__ void noise_fill_kernel(float* x, const Span* spans, float v) {
  const Span sp = spans[blockIdx.y];
  for (long long i = blockIdx.x * (long long)kThreads + threadIdx.x; i < sp.count; i += (long long)gridDim.x * kThreads)
    x[sp.offset + i] = v;
}

// Dropout multiplier of element (t, b, f) of a [T, B, F] batch: bit f % 128 of the Philox draw keyed by (seed; t,
// global utterance offset + b, update, tag | f / 128) -> 0 or 2.  in null: the multiplier itself; in may be out.
__global__ void __launch_bounds__(kThreads) dropout_kernel(const float* in, float* out, long long n, int B, int F,
                                                           unsigned long long seed, unsigned long long update,
                                                           long long utt_offset) {
  const uint2 key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
  for (long long i = blockIdx.x * (long long)kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
    const long long r = i / F, t = r / B;
    const unsigned f = (unsigned)(i - r * F);
    const uint4 ctr = make_uint4((unsigned)t, (unsigned)(utt_offset + (r - t * B)), (unsigned)update, kTagDropout | (f >> 7));
    const uint4 w = curand_Philox4x32_10(ctr, key);
    const unsigned q = (f >> 5) & 3u;
    const unsigned word = q == 0 ? w.x : q == 1 ? w.y : q == 2 ? w.z : w.w;
    const float mult = ((word >> (f & 31u)) & 1u) ? 2.f : 0.f;
    out[i] = in ? in[i] * mult : mult;
  }
}

// One parameter of the weight noise: its flat span and whether it is a subject (the attention's parameters are not)
struct RegSpan { long long offset, count; int subject; };

// mean null: eps of the subjects, 0 elsewhere (replay); else noisy = mean + level eps over the subjects, mean elsewhere.
// The padding between parameters is not written.
__global__ void __launch_bounds__(kThreads) weight_noise_kernel(const float* __restrict__ mean, float* __restrict__ out,
                                                                const RegSpan* spans, float level, unsigned long long seed,
                                                                unsigned long long update) {
  const RegSpan sp = spans[blockIdx.y];
  const long long groups = (sp.count + 3) >> 2;
  for (long long gq = blockIdx.x * (long long)kThreads + threadIdx.x; gq < groups; gq += (long long)gridDim.x * kThreads) {
    const long long i0 = sp.offset + 4 * gq;
    float e[4];
    eps4(seed, update, (unsigned long long)i0 >> 2, e, kTagWeightNoise);
    for (int j = 0; j < 4 && 4 * gq + j < sp.count; ++j) {
      if (!mean) out[i0 + j] = sp.subject ? e[j] : 0.f;
      else out[i0 + j] = sp.subject ? fmaf(level, e[j], mean[i0 + j]) : mean[i0 + j];
    }
  }
}

inline dim3 param_grid(const lvsr_model* m) { return dim3(kCtasPerParam, (unsigned)m->params.size()); }
inline const Span* spans_of(const lvsr_model* m) { return static_cast<const Span*>(m->noise.spans); }

int check_index(const lvsr_model* m, int index, int64_t count) {
  LVSR_CHECK(m && m->noise.on, "adaptive noise is off (lvsr_train_set_adaptive_noise)");
  LVSR_CHECK(index >= 0 && index < (int)m->params.size(), "bad parameter index %d", index);
  LVSR_CHECK(count == m->params[index].count, "parameter '%s' holds %lld values, got %lld", m->params[index].name.c_str(),
             (long long)m->params[index].count, (long long)count);
  return 0;
}

}  // namespace

namespace lvsr {

int noise_sample(lvsr_model* m, cudaStream_t st) {
  ProfScope prof("noise", st);
  lvsr_model::Noise& z = m->noise;
  noise_sample_kernel<<<param_grid(m), kThreads, 0, st>>>(m->flat.get(), z.ls2, z.noisy, spans_of(m), z.cfg.seed,
                                                          (unsigned long long)z.update, z.part);
  LVSR_LAUNCH_CHECK();
  double n = 0.0;
  for (const Param& p : m->params) n += (double)p.count;
  const int nparts = kCtasPerParam * (int)m->params.size();
  noise_prior_kernel<<<1, kThreads, 0, st>>>(z.part, nparts, n, z.cfg.model_cost_coefficient / (double)z.cfg.num_examples, z.stats);
  LVSR_LAUNCH_CHECK();
  z.sampled = true;
  return 0;
}

int noise_gradients(lvsr_model* m, float* grads, float gscale, float* gls2, cudaStream_t st, int* nparts) {
  lvsr_model::Noise& z = m->noise;
  LVSR_CHECK(z.sampled, "adaptive noise: no training forward since the last update (its priors form the gradients)");
  ProfScope prof("noise", st);
  noise_grad_kernel<<<param_grid(m), kThreads, 0, st>>>(grads, gls2, m->flat.get(), z.ls2, spans_of(m), z.stats, gscale,
                                                        (float)(z.cfg.model_cost_coefficient / (double)z.cfg.num_examples),
                                                        nparts ? z.norm_part : nullptr);
  LVSR_LAUNCH_CHECK();
  if (nparts) *nparts = kCtasPerParam * (int)m->params.size();
  return 0;
}

int dropout_apply(const DropoutKey& key, const float* in, float* out, int T, int B, int F, cudaStream_t st) {
  ProfScope prof("dropout", st);
  const long long n = (long long)T * B * F;
  dropout_kernel<<<(unsigned)std::min<long long>(4096, (n + kThreads - 1) / kThreads), kThreads, 0, st>>>(
      in, out, n, B, F, key.seed, (unsigned long long)key.update, key.utt_offset);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int weight_noise_sample(lvsr_model* m, cudaStream_t st) {
  ProfScope prof("weight_noise", st);
  const lvsr_model::Reg& r = m->reg;
  weight_noise_kernel<<<param_grid(m), kThreads, 0, st>>>(m->flat.get(), r.noisy.get(),
                                                          static_cast<const RegSpan*>(r.spans.get()), r.level, r.seed,
                                                          (unsigned long long)r.update);
  LVSR_LAUNCH_CHECK();
  return 0;
}

}  // namespace lvsr

extern "C" {

int lvsr_train_set_adaptive_noise(lvsr_model* m, const lvsr_adaptive_noise* cfg) {
  LVSR_CHECK(m, "null model");
  DeviceGuard device_guard(m);
  if (!cfg) {
    LVSR_CUDA_OK(cudaDeviceSynchronize());        // a training call may still read the buffers
    m->noise = lvsr_model::Noise();
    return 0;
  }
  LVSR_CHECK(cfg->init_sigma > 0.0 && std::isfinite(cfg->init_sigma), "adaptive noise: init_sigma must be > 0");
  LVSR_CHECK(cfg->model_cost_coefficient >= 0.0 && std::isfinite(cfg->model_cost_coefficient),
             "adaptive noise: model_cost_coefficient must be >= 0");
  LVSR_CHECK(cfg->num_examples > 0, "adaptive noise: num_examples must be > 0");
  lvsr_model::Noise& z = m->noise;
  const size_t n = (size_t)m->flat_count, np = m->params.size();
  const size_t nparts = (size_t)kCtasPerParam * np;
  LVSR_CUDA_OK(cudaDeviceSynchronize());          // after every call queued on the handle, on any stream
  if (!z.mem) {                                   // both allocations, or neither
    DeviceBuffer<float> mem;
    DeviceBuffer<char> aux;
    LVSR_CUDA_OK(mem.alloc(6 * n * sizeof(float)));
    const size_t span_bytes = (np * sizeof(Span) + 255) & ~(size_t)255;
    LVSR_CUDA_OK(aux.alloc(span_bytes + (4 + 4 * nparts) * sizeof(double) + nparts * sizeof(float)));
    std::vector<Span> h(np);
    for (size_t i = 0; i < np; ++i) h[i] = Span{m->params[i].offset, m->params[i].count};
    LVSR_CUDA_OK(cudaMemcpy(aux.get(), h.data(), np * sizeof(Span), cudaMemcpyHostToDevice));
    z.mem = std::move(mem);
    z.aux = std::move(aux);
    float* p = z.mem.get();
    z.ls2 = p; z.noisy = p + n; z.gls2 = p + 2 * n;
    z.velocity = p + 3 * n; z.ms_step = p + 4 * n; z.ms_dx = p + 5 * n;
    z.spans = z.aux.get();
    z.stats = reinterpret_cast<double*>(z.aux.get() + span_bytes);
    z.part = z.stats + 4;
    z.norm_part = reinterpret_cast<float*>(z.part + 4 * nparts);
  }
  LVSR_CUDA_OK(cudaMemset(z.mem.get(), 0, 6 * n * sizeof(float)));
  LVSR_CUDA_OK(cudaMemset(z.stats, 0, 4 * sizeof(double)));
  // graph.py:173-175: ls2 = log(init_sigma) * 2 / log_sigma_scale, in float32
  noise_fill_kernel<<<param_grid(m), kThreads>>>(z.ls2, spans_of(m), (float)(log(cfg->init_sigma) * 2.0 / kLogSigmaScale));
  LVSR_LAUNCH_CHECK();
  LVSR_CUDA_OK(cudaDeviceSynchronize());
  z.cfg = *cfg;
  z.on = true;
  z.update = 0;
  z.sampled = false;
  return 0;
}

int lvsr_train_get_noise_param(const lvsr_model* m, int index, float* host, int64_t count) {
  if (int rc = check_index(m, index, count)) return rc;
  LVSR_CHECK(host, "null argument");
  DeviceGuard device_guard(m);
  return copy_on_handle(m, host, m->noise.ls2 + m->params[index].offset, (size_t)count * sizeof(float),
                        cudaMemcpyDeviceToHost);
}

int lvsr_train_set_noise_param(lvsr_model* m, int index, const float* host, int64_t count) {
  if (int rc = check_index(m, index, count)) return rc;
  LVSR_CHECK(host, "null argument");
  DeviceGuard device_guard(m);
  if (int rc = copy_on_handle(m, m->noise.ls2 + m->params[index].offset, host, (size_t)count * sizeof(float),
                              cudaMemcpyHostToDevice)) return rc;
  m->noise.sampled = false;
  return 0;
}

int lvsr_train_noise_stats(lvsr_model* m, double out[3]) {
  LVSR_CHECK(m && out, "null argument");
  LVSR_CHECK(m->noise.on, "adaptive noise is off (lvsr_train_set_adaptive_noise)");
  DeviceGuard device_guard(m);
  LVSR_CUDA_OK(cudaDeviceSynchronize());
  LVSR_CUDA_OK(cudaMemcpy(out, m->noise.stats, 3 * sizeof(double), cudaMemcpyDeviceToHost));
  return 0;
}

int lvsr_train_noise_sample(lvsr_model* m, int64_t update, float* eps_dev, void* stream) {
  LVSR_CHECK(m && eps_dev && update >= 0, "train_noise_sample: bad arguments");
  LVSR_CHECK(m->noise.on, "adaptive noise is off (lvsr_train_set_adaptive_noise)");
  DeviceGuard device_guard(m);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_stream(m, st)) return rc;
  ProfScope prof("noise", st);
  LVSR_CUDA_OK(cudaMemsetAsync(eps_dev, 0, (size_t)m->flat_count * sizeof(float), st));
  noise_eps_kernel<<<param_grid(m), kThreads, 0, st>>>(eps_dev, spans_of(m), m->noise.cfg.seed, (unsigned long long)update);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int lvsr_train_noise_params(lvsr_model* m, float* out_dev, void* stream) {
  LVSR_CHECK(m && out_dev, "train_noise_params: null argument");
  LVSR_CHECK(m->noise.on, "adaptive noise is off (lvsr_train_set_adaptive_noise)");
  DeviceGuard device_guard(m);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_stream(m, st)) return rc;
  LVSR_CUDA_OK(cudaMemcpyAsync(out_dev, m->noise.noisy, (size_t)m->flat_count * sizeof(float), cudaMemcpyDeviceToDevice,
                               st));
  return 0;
}

int lvsr_train_noise_gradients(lvsr_model* m, float* grads_dev, float gscale, float* ls2_grads_dev, void* stream) {
  LVSR_CHECK(m && grads_dev && ls2_grads_dev, "train_noise_gradients: null argument");
  LVSR_CHECK(m->noise.on, "adaptive noise is off (lvsr_train_set_adaptive_noise)");
  DeviceGuard device_guard(m);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_stream(m, st)) return rc;
  LVSR_CUDA_OK(cudaMemsetAsync(ls2_grads_dev, 0, (size_t)m->flat_count * sizeof(float), st));
  return noise_gradients(m, grads_dev, gscale, ls2_grads_dev, st, nullptr);
}

int lvsr_train_set_regularization(lvsr_model* m, const lvsr_regularization* cfg) {
  LVSR_CHECK(m, "null model");
  DeviceGuard device_guard(m);
  if (cfg) {
    LVSR_CHECK(cfg->dropout == 0 || cfg->dropout == 1, "regularization: dropout must be 0 or 1");
    LVSR_CHECK(cfg->noise_level >= 0.0 && std::isfinite(cfg->noise_level), "regularization: noise_level must be >= 0");
    LVSR_CHECK(cfg->penalty_coof >= 0.0 && std::isfinite(cfg->penalty_coof), "regularization: penalty_coof must be >= 0");
  }
  if (m->reg.spans || m->reg.penalty) LVSR_CUDA_OK(cudaDeviceSynchronize());     // a training call may still read the buffers
  // the new settings and buffers replace the handle's only once every allocation succeeded
  lvsr_model::Reg r;
  if (!cfg) {
    m->reg = std::move(r);
    return 0;
  }
  r.dropout = cfg->dropout != 0;
  r.level = (float)cfg->noise_level;
  r.seed = cfg->seed ? cfg->seed : 1;
  r.penalty_coof = (float)cfg->penalty_coof;
  if (r.penalty_coof > 0.f) {
    LVSR_CUDA_OK(r.penalty.alloc(sizeof(float)));
    LVSR_CUDA_OK(cudaMemset(r.penalty.get(), 0, sizeof(float)));
  }
  if (r.level > 0.f) {
    // Blocks' apply_noise subjects: every parameter outside Selector(generator.transition.attention) (lvsr/main.py:297)
    const size_t np = m->params.size();
    std::vector<RegSpan> h(np);
    for (size_t i = 0; i < np; ++i) {
      const std::string& name = m->params[i].name;
      const bool attention = name.rfind(std::string(ATT) + "/", 0) == 0 || name.rfind(std::string(CONT) + "/", 0) == 0;
      h[i] = RegSpan{m->params[i].offset, m->params[i].count, attention ? 0 : 1};
    }
    LVSR_CUDA_OK(r.spans.alloc(np * sizeof(RegSpan)));
    LVSR_CUDA_OK(cudaMemcpy(r.spans.get(), h.data(), np * sizeof(RegSpan), cudaMemcpyHostToDevice));
    LVSR_CUDA_OK(r.noisy.alloc((size_t)m->flat_count * sizeof(float)));
    LVSR_CUDA_OK(cudaMemset(r.noisy.get(), 0, (size_t)m->flat_count * sizeof(float)));
  }
  m->reg = std::move(r);
  return 0;
}

int lvsr_train_penalty_sum(lvsr_model* m, float* penalty_dev, void* stream) {
  LVSR_CHECK(m && penalty_dev, "train_penalty_sum: null argument");
  LVSR_CHECK(m->reg.penalty, "the alignment penalty is off (lvsr_train_set_regularization)");
  DeviceGuard device_guard(m);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_stream(m, st)) return rc;
  LVSR_CUDA_OK(cudaMemcpyAsync(penalty_dev, m->reg.penalty.get(), sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

int lvsr_train_set_utterance_offset(lvsr_model* m, int64_t utterance_offset) {
  LVSR_CHECK(m && utterance_offset >= 0, "train_set_utterance_offset: bad arguments");
  m->reg.utt_offset = utterance_offset;        // a kernel argument of the next training forward: no wait needed
  return 0;
}

int lvsr_train_dropout_mask(lvsr_model* m, int64_t update, int64_t utterance_offset, int32_t T, int32_t B, int32_t F,
                            float* mult_dev, void* stream) {
  LVSR_CHECK(m && mult_dev && update >= 0 && utterance_offset >= 0 && T > 0 && B > 0 && F > 0,
             "train_dropout_mask: bad arguments");
  DeviceGuard device_guard(m);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_stream(m, st)) return rc;
  return dropout_apply(DropoutKey{m->reg.seed, update, utterance_offset}, nullptr, mult_dev, T, B, F, st);
}

int lvsr_train_weight_noise_sample(lvsr_model* m, int64_t update, float* eps_dev, void* stream) {
  LVSR_CHECK(m && eps_dev && update >= 0, "train_weight_noise_sample: bad arguments");
  LVSR_CHECK(m->reg.spans, "weight noise is off (lvsr_train_set_regularization)");
  DeviceGuard device_guard(m);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_stream(m, st)) return rc;
  ProfScope prof("weight_noise", st);
  LVSR_CUDA_OK(cudaMemsetAsync(eps_dev, 0, (size_t)m->flat_count * sizeof(float), st));
  weight_noise_kernel<<<param_grid(m), kThreads, 0, st>>>(nullptr, eps_dev, static_cast<const RegSpan*>(m->reg.spans.get()),
                                                          0.f, m->reg.seed, (unsigned long long)update);
  LVSR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
