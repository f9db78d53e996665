// Content + location attention step: one launch = take_glimpses for R decoder rows.
//
// Replaces, for every row, SequenceContentAndConvAttention.take_glimpses
// (lvsr/bricks/attention.py:120-183): window cut, Conv1D of the previous alignment
// (lvsr/expressions.py:28-54, true convolution, centre crop :108-111), energies
// (:98-114), normaliser (:191-213), weighted average (B/bricks/attention.py:235-256)
// and the paste back into [R, T'] (:177-181).
//
// Mapping: a row's P/H slices (T' x (M+E) floats, ~1 MB) are streamed once per
// step; a thread-block CLUSTER of `cs` CTAs splits the window of one row along time,
// each CTA produces a local (max, sum, weighted partial context) triple and the
// cluster combines them through distributed shared memory (online-softmax merge) --
// one cluster barrier per step, no global round trip.  Warp-shuffle reductions for
// the energy dot products and the softmax statistics.
#include "attention_row.cuh"

namespace lvsr {

namespace {

constexpr int ATT_THREADS = ATT_NT;

// ---------------------------------------------------------------------------------
// window kernel
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) window_kernel(WindowArgs a) {
  __shared__ float s_lo[8], s_hi[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int sg = blockIdx.x;                              // one CTA per segment
  const int r_begin = a.seg_start ? a.seg_start[sg] : 0, r_end = a.seg_start ? a.seg_start[sg + 1] : a.R;
  const int Tp = a.Tp;                                    // row pitch of the weights
  const int Tl = a.seg_len ? a.seg_len[sg] : Tp;          // `length` of the reference: the utterance's own encoded length
  if (a.prior.type == LVSR_PRIOR_EXPANDING) {
    // lvsr/bricks/attention.py:127-132 -- step[0] (first row of the batch) decides for the whole batch
    if (tid == 0) {
      const double st = (double)((a.step ? a.step[r_begin] : 0LL) + a.step_offset);
      double begin = a.prior.initial_begin + st * a.prior.min_speed;
      double end = a.prior.initial_end + st * a.prior.max_speed;
      begin = fmax(0.0, fmin((double)(Tl - 1), begin));
      end = fmax(0.0, fmin((double)Tl, end));
      a.win[2 * sg] = (int)floor(begin);
      a.win[2 * sg + 1] = (int)ceil(end);
    }
    for (int r = r_begin + tid; r < r_end; r += blockDim.x) {
      a.lohi[2 * r] = -1e30f;
      a.lohi[2 * r + 1] = 1e30f;
    }
    return;
  }
  float my_lo = 1e30f, my_hi = -1e30f;
  const int chunk = (Tl + 31) / 32;
  for (int r = r_begin + warp; r < r_end; r += 8) {
    const float* w = a.weights + (long long)r * Tp;
    const int i0 = lane * chunk, i1 = min(Tl, i0 + chunk);
    double pos;
    if (a.prior.type == LVSR_PRIOR_WINDOW_MEAN) {
      double acc = 0.0;                                   // :136-137
      for (int i = i0; i < i1; ++i) acc += (double)w[i] * (double)i;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      pos = acc;
    } else {
      // window_around_median, :138-144: first index j* with cumsum >= 0.5; the reference's
      // argmax of the shifted difference gives j* - 1 (0 when j* == 0 or no crossing)
      double part = 0.0;
      for (int i = i0; i < i1; ++i) part += (double)w[i];
      double incl = part;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        double n = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += n;
      }
      double run = incl - part;
      int cross = 0x7fffffff;
      for (int i = i0; i < i1; ++i) {
        run += (double)w[i];
        if (run - 0.5 >= 0.0) { cross = i; break; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) cross = min(cross, __shfl_xor_sync(0xffffffffu, cross, o));
      pos = (cross == 0x7fffffff || cross == 0) ? 0.0 : (double)(cross - 1);
    }
    const float lo = (float)floor(pos - a.prior.before);   // :146-147
    const float hi = (float)ceil(pos + a.prior.after);
    if (lane == 0) {
      a.lohi[2 * r] = lo;
      a.lohi[2 * r + 1] = hi;
    }
    my_lo = fminf(my_lo, lo);
    my_hi = fmaxf(my_hi, hi);
  }
  if (lane == 0) { s_lo[warp] = my_lo; s_hi[warp] = my_hi; }
  __syncthreads();
  if (tid == 0) {
    float lo = s_lo[0], hi = s_hi[0];
    for (int i = 1; i < 8; ++i) { lo = fminf(lo, s_lo[i]); hi = fmaxf(hi, s_hi[i]); }
    a.win[2 * sg] = (int)fmaxf(0.f, lo);                    // :149-150
    a.win[2 * sg + 1] = (int)fminf((float)Tl, hi);
  }
}

// ---------------------------------------------------------------------------------
// attention step kernel: one cluster of `cs` CTAs per decoder row
// ---------------------------------------------------------------------------------
template <bool LOC>
__device__ __forceinline__ void att_step_row(const AttStepArgs& a, int tc_cap) {
  extern __shared__ __align__(16) float smem[];
  cg::cluster_group cluster = cg::this_cluster();
  const int cs = (int)cluster.num_blocks();
  const int rank = (int)cluster.block_rank();
  const int row = blockIdx.x / cs;
  // arrive now, wait just before the first remote write: guarantees every CTA of the
  // cluster is resident without stalling the prologue
  asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
  AttRowIO io;
  io.P = a.P; io.H = a.H; io.maskH = a.maskH;
  io.q_row = a.q + (long long)row * a.M;
  io.w_prev = a.w_prev + (long long)row * a.Tp;
  io.filt = a.filt; io.Wh = a.Wh; io.v = a.v; io.v_bias = a.v_bias;
  io.w_out = a.w_out + (long long)row * a.Tp;
  io.e_out = a.e_out + (long long)row * a.Tp;
  io.ctx_out = a.ctx + (long long)row * a.E;
  io.u = a.row_utt ? a.row_utt[row] : row;
  io.U = a.U; io.Tp = a.Tp; io.M = a.M; io.E = a.E; io.K = a.K; io.n = a.n; io.normalizer = a.normalizer;
  const int sg = a.row_seg ? a.row_seg[row] : 0;
  io.b0 = a.win[2 * sg]; io.b1 = a.win[2 * sg + 1];
  io.lo = a.lohi[2 * row]; io.hi = a.lohi[2 * row + 1];
  attention_row<false, LOC>(io, smem, tc_cap, rank, cs, false, false, true);
}

__global__ void __launch_bounds__(ATT_THREADS, 1) att_step_kernel(AttStepArgs a, int tc_cap) { att_step_row<true>(a, tc_cap); }

// content-only attention (SequenceContentAttention.take_glimpses, B/bricks/attention.py:370-388)
__global__ void __launch_bounds__(ATT_THREADS, 1) att_content_step_kernel(AttStepArgs a, int tc_cap) {
  att_step_row<false>(a, tc_cap);
}

int num_sms() { return device_sm_count(); }

constexpr size_t ATT_SMEM_MAX = 227 * 1024;   // dynamic shared memory one CTA may opt in to on sm_90

// Dynamic shared memory (bytes) of one attention-step CTA when clusters of cs CTAs split a row of T' positions.
size_t att_step_smem(const AttStepArgs& a, bool loc, int cs) {
  const int tc_cap = ceil_div(a.Tp, cs);
  return (loc ? att_smem_floats(a.M, a.E, a.K, a.n, tc_cap, cs) : att_smem_floats<false>(a.M, a.E, 0, 0, tc_cap, cs)) *
         sizeof(float);
}

int launch_att(const AttStepArgs& a, bool loc, int cs, size_t smem, cudaStream_t stream) {
  const int tc_cap = ceil_div(a.Tp, cs);
  static size_t configured[2][LVSR_MAX_DEVICES] = {{0}};
  const int dev = current_device();
  void (*kernel)(AttStepArgs, int) = loc ? att_step_kernel : att_content_step_kernel;
  if (smem > configured[loc][dev]) {
    LVSR_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured[loc][dev] = smem;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(a.R * cs);
  cfg.blockDim = dim3(ATT_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  LVSR_CUDA_OK(cudaLaunchKernelEx(&cfg, kernel, a, tc_cap));
  g_launch_count++;
  return 0;
}

}  // namespace

int attention_window(const WindowArgs& a, cudaStream_t stream) {
  ProfScope prof("window", stream);
  window_kernel<<<a.seg_start ? a.nseg : 1, 256, 0, stream>>>(a);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int attention_step(const AttStepArgs& a, bool location, int* cs_out, cudaStream_t stream) {
  ProfScope prof("attention", stream);
  LVSR_CHECK(a.M == 128 || a.M == 256 || a.M == 512, "attention_step: dim_matcher %d unsupported (128, 256 or 512)", a.M);
  LVSR_CHECK(a.E % 4 == 0 && a.E <= 4 * ATT_NT, "attention_step: encoded dim must be a multiple of 4 and <= %d", 4 * ATT_NT);
  LVSR_CHECK(a.E / 4 <= ATT_THREADS, "attention_step: encoded dim %d > 1024 unsupported", a.E);
  LVSR_CHECK(!location || (a.K >= 1 && a.K <= 16), "attention_step: conv_num_filters %d not in [1,16]", a.K);
  if (a.R <= 0) return 0;
  // cluster size: split a row's window over as many CTAs as keeps R*cs within one wave
  int cs = 1;
  const int sms = num_sms();
  while (cs < 8 && a.R * cs * 2 <= sms && ceil_div(a.Tp, cs * 2) >= 16) cs *= 2;
  // a row longer than one CTA's shared memory holds is split further.  Clusters of one step never wait for each other,
  // so the grid need not be co-resident and a larger cluster than one wave allows always runs.
  while (cs < 8 && att_step_smem(a, location, cs) > ATT_SMEM_MAX && ceil_div(a.Tp, cs * 2) >= 16) cs *= 2;
  // LVSR_ATT_CS=1|2|4|8 (DESIGN §7, read on every call) replaces the choice above when the forced size keeps
  // ceil(T'/cs) >= 16 and its shared memory fits; otherwise it is declined.
  if (const char* s = getenv("LVSR_ATT_CS")) {
    const int f = atoi(s);
    LVSR_CHECK(f == 1 || f == 2 || f == 4 || f == 8, "LVSR_ATT_CS=%s: expected 1, 2, 4 or 8", s);
    if ((f == 1 || ceil_div(a.Tp, f) >= 16) && att_step_smem(a, location, f) <= ATT_SMEM_MAX) cs = f;
  }
  const size_t smem = att_step_smem(a, location, cs);
  LVSR_CHECK(smem <= ATT_SMEM_MAX,
             "attention_step: T'=%d positions do not fit in shared memory at any cluster size: %zu B per CTA in "
             "clusters of %d (M=%d, E=%d, conv_num_filters=%d, conv_n=%d) exceeds the 227 KB limit",
             a.Tp, smem, cs, a.M, a.E, location ? a.K : 0, location ? a.n : 0);
  *cs_out = cs;
  return launch_att(a, location, cs, smem, stream);
}

}  // namespace lvsr
