// Shared helpers for the sm_90a kernels of the attention-lvcsr hot path.
#pragma once
#include <cuda_runtime.h>
#include <cooperative_groups.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <string>
#include <utility>

namespace lvsr {

namespace cg = cooperative_groups;

extern thread_local std::string g_last_error;
extern long long g_launch_count;
extern std::atomic<long long> g_device_bytes;    // bytes every DeviceBuffer holds (lvsr_device_bytes)

int set_error(const char* fmt, ...);

// Optional per-launch CUDA-event timing (see lvsr_profile_enable in include/lvsr_b200.h).
struct ProfScope {
  int slot;
  cudaStream_t st;
  ProfScope(const char* kernel_class, cudaStream_t stream);
  ~ProfScope();
};

#define LVSR_CUDA_OK(expr)                                                          \
  do {                                                                              \
    cudaError_t _e = (expr);                                                        \
    if (_e != cudaSuccess)                                                          \
      return ::lvsr::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                               __FILE__, __LINE__);                                 \
  } while (0)

#define LVSR_CHECK(cond, ...)                          \
  do {                                                 \
    if (!(cond)) return ::lvsr::set_error(__VA_ARGS__); \
  } while (0)

#define LVSR_LAUNCH_CHECK()                                                         \
  do {                                                                              \
    ::lvsr::g_launch_count++;                                                       \
    cudaError_t _e = cudaGetLastError();                                            \
    if (_e != cudaSuccess)                                                          \
      return ::lvsr::set_error("kernel launch failed: %s (%s:%d)",                  \
                               cudaGetErrorString(_e), __FILE__, __LINE__);         \
  } while (0)

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// The owner of one cudaMalloc allocation, and the only code that calls cudaMalloc / cudaFree: move-only, freed when it
// is destroyed, reset or assigned to.  Releasing never waits: code that drops a buffer enqueued work may still read
// waits for that work first.
template <class T>
class DeviceBuffer {
 public:
  DeviceBuffer() = default;
  DeviceBuffer(DeviceBuffer&& o) noexcept : p_(std::exchange(o.p_, nullptr)), bytes_(std::exchange(o.bytes_, 0)) {}
  DeviceBuffer& operator=(DeviceBuffer&& o) noexcept {
    if (this != &o) {
      reset();
      p_ = std::exchange(o.p_, nullptr);
      bytes_ = std::exchange(o.bytes_, 0);
    }
    return *this;
  }
  ~DeviceBuffer() { reset(); }

  // Replaces the buffer by `bytes` of device memory (empty when the allocation fails)
  cudaError_t alloc(size_t bytes) {
    reset();
    void* p = nullptr;
    const cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) return e;
    p_ = static_cast<T*>(p);
    bytes_ = bytes;
    g_device_bytes += (long long)bytes;
    return cudaSuccess;
  }
  // At least `bytes`: a smaller buffer is replaced once `stream`, whose work may still read it, has drained
  cudaError_t grow(size_t bytes, cudaStream_t stream) {
    if (bytes <= bytes_) return cudaSuccess;
    if (p_) {
      const cudaError_t e = cudaStreamSynchronize(stream);
      if (e != cudaSuccess) return e;
    }
    return alloc(bytes);
  }
  void reset() {
    if (!p_) return;
    cudaFree(p_);
    g_device_bytes -= (long long)bytes_;
    p_ = nullptr;
    bytes_ = 0;
  }
  T* get() const { return p_; }
  size_t bytes() const { return bytes_; }
  explicit operator bool() const { return p_ != nullptr; }

 private:
  T* p_ = nullptr;
  size_t bytes_ = 0;
};

// Every entry point runs on its handle's GPU (the device current when the handle was created), whatever device the
// calling thread has current.  Handle: lvsr_model or lvsr_frontend; a null handle switches nothing.
struct DeviceGuard {
  int prev = -1;
  template <class Handle>
  explicit DeviceGuard(const Handle* h) {
    int cur = 0;
    if (h && cudaGetDevice(&cur) == cudaSuccess && cur != h->device) {
      prev = cur;
      cudaSetDevice(h->device);
    }
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// Every entry point that takes a stream binds it first, before it sizes a workspace or touches per-handle device
// state: a call on another stream than the handle's last one first waits for everything the handle enqueued there, so
// two streams never share its workspaces, status words or parameters at once.
template <class Handle>
static inline int bind_stream(Handle* h, cudaStream_t st) {
  LVSR_CHECK(h != nullptr, "null model");
  if (st != h->stream) {
    LVSR_CUDA_OK(cudaStreamSynchronize(h->stream));
    h->stream = st;
  }
  return 0;
}

// Function attributes (dynamic shared-memory opt-in), SM counts and occupancy answers are properties
// of a DEVICE, not of the process: caches are keyed by the current device ordinal.
constexpr int LVSR_MAX_DEVICES = 64;
static inline int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return (dev >= 0 && dev < LVSR_MAX_DEVICES) ? dev : 0;
}
static inline int device_sm_count() {
  static int sms[LVSR_MAX_DEVICES] = {0};
  const int dev = current_device();
  if (sms[dev] == 0) {
    cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
    if (sms[dev] <= 0) sms[dev] = 132;
  }
  return sms[dev];
}

// Two N(0, 1) draws from two 32-bit Philox words, Box-Muller in fp32 (the weight noise's and the front end's dither)
__device__ __forceinline__ float2 box_muller(unsigned x, unsigned y) {
  const float u = ((float)(x >> 8) + 0.5f) * (1.f / 16777216.f);    // (0, 1): log(u) is finite
  const float v = (float)(y >> 8) * (1.f / 16777216.f);
  const float r = sqrtf(-2.f * logf(u));
  float s, c;
  sincospif(2.f * v, &s, &c);
  return make_float2(r * c, r * s);
}

// ---- device math: accurate enough for the 1e-4 gate against the float64 oracle ----
__device__ __forceinline__ float sigmoidf_acc(float x) { return 1.0f / (1.0f + __expf(-x)); }

// tanh via exp: |err| ~ 1e-7 absolute, which is what energies / states need.
__device__ __forceinline__ float tanhf_acc(float x) {
  float ax = fabsf(x);
  if (ax < 0.04f) {  // odd Taylor polynomial keeps RELATIVE accuracy near 0
    float x2 = x * x;
    return x * (1.0f + x2 * (-0.33333333f + x2 * 0.13333334f));
  }
  float e = __expf(-2.0f * ax);
  float t = (1.0f - e) / (1.0f + e);
  return copysignf(t, x);
}

// 2-MUFU activations (ex2 + rcp): |abs err| ~ 2e-7; saturate correctly at +-inf.
// On the flush-to-zero forms of ex2 / rcp: `__expf` / `__fdividef` wrap every MUFU in a subnormal range fix-up
// (FSETP + two predicated FMULs) and cannot fold the scale of the argument -- 10 instructions per tanh instead of 5,
// in the decoder's energy loop (8 M tanh per step) and on the critical chain of every recurrent step.  A flushed exp only
// matters beyond |x| ~ 87 (43 for tanh), where the result is 0 / +-1 to 1e-38 either way.
__device__ __forceinline__ float ex2_ftz(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_ftz(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_sigmoid(float x) { return rcp_ftz(1.0f + ex2_ftz(-1.4426950408889634f * x)); }
__device__ __forceinline__ float fast_tanh(float x) { return fmaf(-2.0f, rcp_ftz(1.0f + ex2_ftz(2.8853900817779268f * x)), 1.0f); }


// ---- data-flow synchronisation: the data IS the flag ----------------------------------------
// Buffers that carry values between CTAs of a persistent kernel are pre-filled with a sentinel
// bit pattern (all ones: a NaN no arithmetic produces) and are written exactly once per element.
// A consumer simply re-reads an element until it is no longer the sentinel: one store plus one
// load on the critical path instead of store -> fence -> flag -> poll -> load.
constexpr unsigned LVSR_SENTINEL = 0xFFFFFFFFu;
constexpr unsigned LVSR_SPIN_LIMIT = 1u << 22;
// Launch status word of a data-flow kernel (device memory, zeroed by the host before the launch):
//   0 ok; LVSR_FLOW_TIMEOUT: a value never arrived (every poller gives up, the kernel runs to its
//   end with meaningless data instead of trapping -- a trap would take the whole CUDA context and
//   PyTorch with it); LVSR_FLOW_BAD_CLUSTER: the launch did not get the planned cluster shape.
// The host reads it at its next synchronisation point and re-runs the call on the step-wise kernels.
enum { LVSR_FLOW_OK = 0, LVSR_FLOW_TIMEOUT = 2, LVSR_FLOW_BAD_CLUSTER = 3 };
static __constant__ unsigned g_flow_spin_limit = LVSR_SPIN_LIMIT;
static __constant__ unsigned* g_flow_status = nullptr;
__device__ __forceinline__ void st_flow_f32(float* p, float v) {
  asm volatile("st.relaxed.gpu.global.f32 [%0], %1;\n" ::"l"(p), "f"(v) : "memory");
}
// Called every 1024 unsuccessful polls: true = stop waiting (this or another poller timed out).
static __device__ __noinline__ bool flow_give_up(unsigned spins) {
  unsigned* st = g_flow_status;
  if (st == nullptr) {
    if (spins > g_flow_spin_limit) __trap();
    return false;
  }
  if (spins > g_flow_spin_limit) atomicCAS(st, 0u, (unsigned)LVSR_FLOW_TIMEOUT);
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(st) : "memory");
  return v != 0u;
}
__device__ __forceinline__ float ld_flow_f32(const float* p) {
  unsigned v, spins = 0;
  while (true) {
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
    if (v != LVSR_SENTINEL) break;
    if (((++spins) & 1023u) == 0u && flow_give_up(spins)) { v = 0u; break; }
  }
  return __uint_as_float(v);
}
// One attempt, no spinning: issue several of these back to back, then validate with flow_ready()
// and fall back to ld_flow_f4 for the (rare) values that had not arrived.
__device__ __forceinline__ float4 ld_relaxed_f4(const float* p) {
  unsigned x, y, z, w;
  asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];\n"
               : "=r"(x), "=r"(y), "=r"(z), "=r"(w)
               : "l"(p)
               : "memory");
  return make_float4(__uint_as_float(x), __uint_as_float(y), __uint_as_float(z), __uint_as_float(w));
}
__device__ __forceinline__ bool flow_ready(const float4& v) {
  return __float_as_uint(v.x) != LVSR_SENTINEL && __float_as_uint(v.y) != LVSR_SENTINEL &&
         __float_as_uint(v.z) != LVSR_SENTINEL && __float_as_uint(v.w) != LVSR_SENTINEL;
}
__device__ __forceinline__ float4 ld_flow_f4(const float* p) {
  unsigned x, y, z, w, spins = 0;
  while (true) {
    asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];\n"
                 : "=r"(x), "=r"(y), "=r"(z), "=r"(w)
                 : "l"(p)
                 : "memory");
    if (x != LVSR_SENTINEL && y != LVSR_SENTINEL && z != LVSR_SENTINEL && w != LVSR_SENTINEL) break;
    if (((++spins) & 1023u) == 0u && flow_give_up(spins)) { x = y = z = w = 0u; break; }
  }
  return make_float4(__uint_as_float(x), __uint_as_float(y), __uint_as_float(z), __uint_as_float(w));
}

// fp32 pair arithmetic: two independent FFMA chains (even k in .x, odd k in .y), summed once at the end.
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
__device__ __forceinline__ float sum2(float2 v) { return v.x + v.y; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Reduce N per-lane partial sums across lanes with a halving exchange over the lane-index bits
// 16, 8, ... down to OMIN (OMIN = 1: all 32 lanes; OMIN = 4: the 8 lanes that differ in bits 2..4,
// i.e. four independent groups per warp).  After the call acc[0 .. max(1, N / lanes)) hold fully
// reduced values and the returned base says which: acc[j] == sum over the group of original
// acc[base + j].  When N < lanes the tail stages are plain butterflies: lane groups hold duplicates.
template <int NTOT, int n, int o, int OMIN>
__device__ __forceinline__ void rs_stage(float (&acc)[NTOT], int lane, int& base) {
  if constexpr (o >= OMIN && o > 0) {
    if constexpr (n > 1) {
      constexpr int h = n / 2;
      const bool up = (lane & o) != 0;
#pragma unroll
      for (int j = 0; j < h; ++j) {
        float mine = up ? acc[j + h] : acc[j];
        float theirs = up ? acc[j] : acc[j + h];
        acc[j] = mine + __shfl_xor_sync(0xffffffffu, theirs, o);
      }
      if (up) base += h;
      rs_stage<NTOT, h, o / 2, OMIN>(acc, lane, base);
    } else {
      acc[0] += __shfl_xor_sync(0xffffffffu, acc[0], o);
      rs_stage<NTOT, 1, o / 2, OMIN>(acc, lane, base);
    }
  }
}
template <int N, int OMIN = 1>
__device__ __forceinline__ int warp_reduce_scatter(float (&acc)[N], int lane) {
  int base = 0;
  rs_stage<N, N, 16, OMIN>(acc, lane, base);
  return base;
}

// The index base warp_reduce_scatter<N, OMIN> will return for this lane (pure function of lane).
template <int N, int OMIN = 1>
__device__ __forceinline__ int rs_base(int lane) {
  int base = 0, n = N;
#pragma unroll
  for (int o = 16; o >= OMIN && o > 0; o >>= 1) {
    if (n > 1) {
      n >>= 1;
      if (lane & o) base += n;
    }
  }
  return base;
}

}  // namespace lvsr
