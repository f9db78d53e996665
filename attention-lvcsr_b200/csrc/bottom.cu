// The bottom MLP in front of the encoder: SpeechBottom's MLP (lvsr/bricks/recognizer.py:105-157), one Linear and one
// activation per entry of config['net']['bottom']['dims'], applied to every frame.
//
// Forward, per layer: the projection GEMM over the T*B frames (projection_gemm: fp16 head/tail wgmma when the
// contraction is a multiple of 64, 3xTF32 when the packed form exists otherwise, FFMA tiles for the rest), then the
// activation in place.  Backward (train.cu): dZ = dY * act'(Y) from the stored output, then the weight, bias and input
// gradients on the products the encoder's fork weights use.
#include <algorithm>

#include "model.h"

namespace lvsr {

namespace {

// Rectifier = switch(x > 0, x, 0) (libs/blocks/blocks/bricks/simple.py), so its derivative at 0 is 0; Tanh.
template <int ACT>
__device__ __forceinline__ float bottom_act(float x) {
  if (ACT == LVSR_ACT_RELU) return x > 0.f ? x : 0.f;
  return tanhf(x);
}
// derivative from the output y = act(x): relu y > 0 exactly where x > 0; tanh 1 - y^2
template <int ACT>
__device__ __forceinline__ float bottom_act_grad(float y, float dy) {
  if (ACT == LVSR_ACT_RELU) return y > 0.f ? dy : 0.f;
  return dy * (1.f - y * y);
}

// y[0, n) = act(y) in place: float4 over the first n - n % 4 floats (the arena hands out 256-byte aligned buffers),
// the last n % 4 one by one, so that any width works
template <int ACT>
__global__ void __launch_bounds__(256) bottom_act_kernel(float* __restrict__ y, long long n) {
  const long long n4 = n >> 2, stride = (long long)gridDim.x * blockDim.x;
  float4* y4 = reinterpret_cast<float4*>(y);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 v = y4[i];
    v.x = bottom_act<ACT>(v.x); v.y = bottom_act<ACT>(v.y); v.z = bottom_act<ACT>(v.z); v.w = bottom_act<ACT>(v.w);
    y4[i] = v;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long long i = (n4 << 2) + threadIdx.x;
    y[i] = bottom_act<ACT>(y[i]);
  }
}

template <int ACT>
__global__ void __launch_bounds__(256) bottom_act_bwd_kernel(float* __restrict__ dy, const float* __restrict__ y,
                                                             long long n) {
  const long long n4 = n >> 2, stride = (long long)gridDim.x * blockDim.x;
  float4* d4 = reinterpret_cast<float4*>(dy);
  const float4* y4 = reinterpret_cast<const float4*>(y);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = y4[i];
    float4 d = d4[i];
    d.x = bottom_act_grad<ACT>(v.x, d.x); d.y = bottom_act_grad<ACT>(v.y, d.y);
    d.z = bottom_act_grad<ACT>(v.z, d.z); d.w = bottom_act_grad<ACT>(v.w, d.w);
    d4[i] = d;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long long i = (n4 << 2) + threadIdx.x;
    dy[i] = bottom_act_grad<ACT>(y[i], dy[i]);
  }
}

inline int act_grid(long long n) {
  return (int)std::min<long long>(4 * device_sm_count(), std::max<long long>(1, ((n >> 2) + 255) / 256));
}

}  // namespace

size_t bottom_ws_bytes(const lvsr_model* m, int rows) {
  size_t total = 0;
  for (int i = 0; i < m->bottom.num_layers; ++i)
    total += ((size_t)rows * m->bottom.dims[i] + (size_t)2 * rows * gemm_tc_kpad(bottom_input_dim(m, i))) * sizeof(float) +
             1024;
  return total;
}

int bottom_forward(lvsr_model* m, Arena& ws, const float* x, int rows, const float** out, cudaStream_t st) {
  const lvsr_bottom_config& b = m->bottom;
  ProfScope prof("bottom", st);
  const float* cur = x;
  for (int i = 0; i < b.num_layers; ++i) {
    const int din = bottom_input_dim(m, i), dout = b.dims[i];
    float* y = ws.f32((size_t)rows * dout);
    LVSR_CHECK(y, "out of device memory (bottom MLP)");
    {
      ArenaMark mark{ws};      // the split scratch is dead once the GEMM is enqueued (stream order)
      const std::string lin = bottom_linear(i);
      if (int rc = projection_gemm(ws, cur, rows, din, m->P(lin + ".W"), m->use_tc ? &m->bottom_tc[i] : nullptr, dout,
                                   m->P(lin + ".b"), y, st))
        return rc;
    }
    const long long n = (long long)rows * dout;
    if (b.activation == LVSR_ACT_RELU)
      bottom_act_kernel<LVSR_ACT_RELU><<<act_grid(n), 256, 0, st>>>(y, n);
    else
      bottom_act_kernel<LVSR_ACT_TANH><<<act_grid(n), 256, 0, st>>>(y, n);
    LVSR_LAUNCH_CHECK();
    out[i] = y;
    cur = y;
  }
  return 0;
}

int bottom_act_backward(float* dY, const float* Y, long long n, int activation, cudaStream_t st) {
  if (activation == LVSR_ACT_RELU)
    bottom_act_bwd_kernel<LVSR_ACT_RELU><<<act_grid(n), 256, 0, st>>>(dY, Y, n);
  else
    bottom_act_bwd_kernel<LVSR_ACT_TANH><<<act_grid(n), 256, 0, st>>>(dY, Y, n);
  LVSR_LAUNCH_CHECK();
  return 0;
}

}  // namespace lvsr
