// Internal model object behind the opaque lvsr_model handle of include/lvsr_b200.h, shared by the
// inference orchestration (api.cu) and the training step (train.cu).
#pragma once
#include <map>
#include <string>
#include <vector>

#include "kernels.h"
#include "lvsr_b200.h"

namespace lvsr {

// Stack-style device workspace.  Top-level API calls bump-allocate from one block; when
// the block is too small the overflow is served by separate cudaMallocs and the block is
// regrown at the end of the call, so a steady-state workload never allocates.  The arena is
// rewound when a call returns while its kernels may still be in flight: safe because every call
// on the handle runs on the handle's bound stream (bind_stream, common.cuh).
struct Arena {
  DeviceBuffer<char> block;         // base = block + shift (LVSR_WS_SHIFT_KB, read by reserve: placement experiments)
  char* base = nullptr;
  size_t cap = 0, off = 0, overflow_bytes = 0, shift = 0;
  int depth = 0;
  std::vector<DeviceBuffer<char>> overflow;

  void* alloc(size_t bytes) {
    bytes = (bytes + 255) & ~(size_t)255;
    if (off + bytes <= cap) {
      void* p = base + off;
      off += bytes;
      return p;
    }
    DeviceBuffer<char> p;
    if (p.alloc(bytes) != cudaSuccess) return nullptr;
    overflow.push_back(std::move(p));
    overflow_bytes += bytes;
    return overflow.back().get();
  }
  float* f32(size_t n) { return static_cast<float*>(alloc(n * sizeof(float))); }
  long long* i64(size_t n) { return static_cast<long long*>(alloc(n * sizeof(long long))); }
  int* i32(size_t n) { return static_cast<int*>(alloc(n * sizeof(int))); }

  // Grow the block up front (only legal while nothing is allocated from it).
  void reserve(size_t bytes, cudaStream_t stream) {
    if (off != 0 || bytes <= cap) return;
    if (cudaStreamSynchronize(stream) != cudaSuccess) return;
    shift = getenv("LVSR_WS_SHIFT_KB") ? (size_t)atoll(getenv("LVSR_WS_SHIFT_KB")) * 1024 : 0;
    replace(bytes);
  }
  void enter() { depth++; }
  // returns non-zero on CUDA failure
  int leave(cudaStream_t stream) {
    depth--;
    if (depth > 0) return 0;
    const size_t used = off;
    off = 0;
    if (!overflow.empty()) {
      if (cudaStreamSynchronize(stream) != cudaSuccess) return 1;
      overflow.clear();
      replace((size_t)((used + overflow_bytes) * 1.25) + (1 << 20));
      overflow_bytes = 0;
    }
    return 0;
  }
  // a new block of cap `bytes` (0 when the allocation fails)
  void replace(size_t bytes) {
    block.reset();
    base = nullptr;
    cap = 0;
    if (block.alloc(bytes + shift) == cudaSuccess) { cap = bytes; base = block.get() + shift; }
    else cudaGetLastError();
  }
};

// One projection's weights [K, N] packed for the tensor-core GEMM, K-major: fp16 head / tail planes [N, K] with the
// exponent of every column (K a multiple of 64), else tf32 hi / lo planes [N, gemm_tc_kpad(K)].  mem == null: the
// shape has no tensor-core form.
struct TcWeights {
  DeviceBuffer<char> mem;                           // the one allocation the planes below live in
  __half *head = nullptr, *tail = nullptr;
  int* ew = nullptr;
  float *hi = nullptr, *lo = nullptr;
};

struct Param {
  std::string name;
  int64_t shape[2];
  int ndim;
  int64_t count;
  int64_t offset;          // position in the flat parameter / gradient / optimizer-state buffers (floats)
  float* dev;              // = lvsr_model::flat + offset
};

}  // namespace lvsr

using namespace lvsr;

struct lvsr_model {
  lvsr_config cfg;
  lvsr_bottom_config bottom = {};   // the bottom MLP in front of the encoder (num_layers 0: none)
  lvsr_readout_config readout = {}; // the readout's post-merge depth and widths (read through readout_depth / _dim)
  int device = 0;                   // the GPU this handle lives on (current device at lvsr_model_create)
  int ndir = 2;                     // encoder directions: 2 bidirectional, 1 forward only (read through encoder_dirs)
  int E;
  std::vector<Param> params;
  std::map<std::string, int> index;
  // ONE allocation for all parameters, each at a 256-byte aligned offset (padding stays zero): the
  // gradient buffer, the optimizer state and the all-reduce of the training step use the same layout
  DeviceBuffer<float> flat;
  int64_t flat_count = 0;
  // packed, kernel-side weights (rebuilt by finalize)
  std::vector<DeviceBuffer<float>> Wcat, bcat;   // per encoder layer: [Din, 3 ndir D], [3 ndir D] (encoder_fork)
  // the packed inputs of decoder layer l < dec_stack (finalize), gate columns first (update | reset), then the
  // candidate inputs; the parameters of layer l > 0 carry the suffix "#l" (layer_suffix)
  struct DecLayer {
    DeviceBuffer<float> Wd;         // [E, 3C]     distribute [fork_gate_inputs | fork_inputs]
    DeviceBuffer<float> Wff;        // [Cfb, 3C]   generator fork (feedback_fork)
    DeviceBuffer<float> bff;        // [3C]
    DeviceBuffer<float> FF;         // [(V+1), 3C] = feedback . Wff + bff
  } dec[2];
  DeviceBuffer<float> Wb1;          // [E+C, 3C] = dec[0].Wd stacked on [state_to_gates | 0] (persistent decoder)
  // dec_stack 2 (finalize; all inside mem): the attention and the readout see the wide state [s0 | s1] through
  // row-stacked weights
  struct Stack {
    DeviceBuffer<float> mem;        // the one allocation of the buffers below
    float* Ws = nullptr;            // [2C, M]   state_trans/transform_states.W ; transform_states#1.W
    float* Wm = nullptr;            // [2C, Cpm] readout/merge/transform_states.W ; transform_states#1.W
    float* h0 = nullptr;            // [2C]      initial_state of both layers
    float* F = nullptr;             // [C, 3C]   recurrentstack/fork_1 [fork_gate_inputs | fork_inputs] (no bias)
  } stack;
  // dense-projection weights as the tensor-core GEMM reads them (wgmma path); empty = SIMT path
  std::vector<TcWeights> Wcat_tc;
  std::vector<TcWeights> bottom_tc; // per bottom layer: linear_<i>.W [d_in, d_out]
  TcWeights Wp_tc;
  bool use_tc = true;
  float v_bias = 0.f;               // host copy of energy_comp/linear.b
  DeviceBuffer<unsigned> status;    // device word: launch status of the data-flow decoder (common.cuh LVSR_FLOW_*)
  bool force_stepwise = false;      // set while a failed persistent launch is re-run on the step-wise kernels
  long long dec_fallbacks = 0;      // how often that happened
  int32_t dec_plan[16] = {0};       // plan of the last lvsr_cost_matrix (lvsr_model_decoder_plan, LVSR_PLAN_* slots)
  int att_cs = 0;                   // cluster size of the last attention_step launch
  int32_t enc_plan[LVSR_MAX_LAYERS][16] = {};   // per layer: lvsr_model_encoder_plan's LVSR_ENC_* slots
  // per layer: 1 when the last encoder forward streamed its projection behind the previous layer's scan
  int32_t enc_overlap[LVSR_MAX_LAYERS] = {};
  DeviceBuffer<int> enc_tiles;      // device [LVSR_MAX_LAYERS][2]: tiles of those projections done beside / after the scan
  DeviceBuffer<int> enc_claims;     // device: ProjStream::claims of every layer, layer l at enc_claims_off[l]
  size_t enc_claims_off[LVSR_MAX_LAYERS] = {};
  int32_t pre_plan[3] = {0, 0, 0};  // last lvsr_preprocess: path (LVSR_ENC_PATH_*), Kpad, operands (LVSR_ENC_OPS_*)
  bool finalized = false;
  // ---- FST language model (lvsr_model_set_lm); lm_off empty: none attached ----
  DeviceBuffer<long long> lm_off;
  DeviceBuffer<int> lm_label, lm_next;
  DeviceBuffer<float> lm_weight;
  int lm_start = 0;
  lvsr_lm_fusion lm_fusion = {};
  DeviceBuffer<unsigned> lm_status;
  // ---- criterion (lvsr_model_set_criterion; read through tle_criterion and initial_output) ----
  lvsr_criterion criterion = {LVSR_CRITERION_LOG_LIKELIHOOD, 0, 0, -1.0};
  DeviceBuffer<unsigned> tle_status;   // device word of tle_matrices, allocated with the first task-loss criterion
  // The stream of the last call that enqueued work on the handle (bind_stream).  Both arenas, the device words above
  // and the parameter and optimizer buffers are only ever touched in this stream's order.
  cudaStream_t stream = nullptr;
  Arena ws;
  // ---- training (train.cu) ----
  Arena tws;                        // tape + backward workspace
  DeviceBuffer<float> opt_velocity, opt_ms_step, opt_ms_dx;   // flat layout, allocated on first use
  DeviceBuffer<float> opt_scratch;  // [1024 partial sums | norm]
  DeviceBuffer<void> opt_desc;      // device copy of the per-parameter table (train::ParamDesc)
  long long burn_in_left = -1;      // BurnIn counter (-1: not started)
  DeviceBuffer<double> clip;        // device train::CLIP_* words of adaptive clipping (empty: off)
  double clip_init[8] = {};         // their values after lvsr_train_set_adaptive_clipping / lvsr_train_reset
  // ---- lvsr_alignment_stats (stats.cu): [finished-CTA count | 256-byte pad | 2 doubles per batch row] ----
  DeviceBuffer<void> align_mem;
  // ---- adaptive weight noise (noise.cu; lvsr_train_set_adaptive_noise) ----
  struct Noise {
    bool on = false;
    lvsr_adaptive_noise cfg = {};
    long long update = 0;           // update counter of the eps draw; advanced by lvsr_train_apply_updates
    bool sampled = false;           // a sample pass ran since the last update (its priors feed the gradients)
    bool stale = false;             // an update left the packed weights un-built (the next training forward packs
                                    // its noisy copy; any other entry point first waits for the update, check_ready)
    DeviceBuffer<float> mem;        // the one allocation of the buffers below (flat layout each, padding zero)
    float* ls2 = nullptr;           // log-variance parameters
    float* noisy = nullptr;         // means + eps * sigma of the current step
    float* gls2 = nullptr;          // gradients, then steps, of ls2
    float *velocity = nullptr, *ms_step = nullptr, *ms_dx = nullptr;   // optimizer state of ls2
    DeviceBuffer<char> aux;         // the one allocation of the tables below
    void* spans = nullptr;          // device [params]: (offset, count) of every parameter, padding excluded
    double* stats = nullptr;        // device [LVSR_NOISE_*]: model cost, prior mean, prior variance, element count
    double* part = nullptr;         // device partial sums of the sample pass
    float* norm_part = nullptr;     // device partial squared norms of the gradient transform
  } noise;
  // ---- dropout and weight noise (noise.cu; lvsr_train_set_regularization) ----
  struct Reg {
    bool dropout = false;
    float level = 0.f;              // weight noise standard deviation (0: off)
    unsigned long long seed = 1;
    long long update = 0;           // update counter of both draws; advanced by lvsr_train_apply_updates
    long long utt_offset = 0;       // global index of the batch's first utterance (dropout key)
    DeviceBuffer<float> noisy;      // flat layout: the means + level * eps of the current step (padding zero)
    DeviceBuffer<void> spans;       // device [params]: (offset, count, subject): 0 for the attention's parameters
    float penalty_coof = 0.f;       // alignment penalty coefficient (0: off)
    DeviceBuffer<float> penalty;    // device: the penalty sum of the last training forward (penalty_coof > 0)
  } reg;

  const Param* param(const std::string& n) const {     // null when the model has no such parameter
    auto it = index.find(n);
    return it == index.end() ? nullptr : &params[it->second];
  }
  float* P(const std::string& n) const { const Param* p = param(n); return p ? p->dev : nullptr; }
};


namespace lvsr {

static const char* const GEN = "/recognizer/generator";
static const char* const TR = "/recognizer/generator/att_trans";
static const char* const ATT = "/recognizer/generator/att_trans/conv_att";
static const char* const CONT = "/recognizer/generator/att_trans/cont_att";

static inline bool content_attention(const lvsr_model* m) { return m->cfg.attention_type == LVSR_ATT_CONTENT; }
// brick path of the attention's parameters
static inline std::string att_base(const lvsr_model* m) { return content_attention(m) ? CONT : ATT; }

// Width of a decoder state row: dec_stack * C ([s0 | s1] with two layers; lvsr_model_create reads dec_stack 0 as 1)
static inline int state_dim(const lvsr_model* m) { return m->cfg.dec_stack * m->cfg.dim_dec; }
// brick path of the decoder GRU of stack level l: "transition", or inside the RecurrentStack "transition_<l>#<l>"
// (RecurrentStack renames its layers, libs/blocks/blocks/bricks/recurrent.py:819-820)
static inline std::string dec_gru(const lvsr_model* m, int level) {
  if (m->cfg.dec_stack == 1) return std::string(TR) + "/transition";
  return std::string(TR) + "/recurrentstack/transition_" + std::to_string(level) + "#" + std::to_string(level);
}

// The readout's post-merge MLP (lvsr_readout_config): depth k, width d_{j+1} of hidden layer j (readout_dim(m, 0) is
// post_merge_dim), the Blocks path of its Linear j, and the floats per row of the hidden layers above h_0
static inline int readout_depth(const lvsr_model* m) { return m->readout.num_layers; }
static inline int readout_dim(const lvsr_model* m, int j) { return m->readout.dims[j]; }
static inline std::string readout_linear(int j) {
  return std::string(GEN) + "/readout/post_merge/mlp/linear_" + std::to_string(j);
}
static inline size_t readout_hidden_floats(const lvsr_model* m) {
  size_t n = 0;
  for (int j = 1; j < readout_depth(m); ++j) n += readout_dim(m, j);
  return n;
}

// Directions of every encoder layer: 2 for Bidirectional, 1 for a forward-only RecurrentWithFork (net.bidir False,
// lvsr/bricks/__init__.py:54-78).  Layer l's output, and layer l + 1's input, is encoder_dirs(m) * dims_bidir[l] wide.
static inline int encoder_dirs(const lvsr_model* m) { return m->ndir; }
static inline int encoder_output_dim(const lvsr_model* m, int l) { return encoder_dirs(m) * m->cfg.dims_bidir[l]; }

// brick path of encoder layer l, direction dir: "bidir<l>/forward|backward", or "with_fork<l>" when unidirectional
static inline std::string enc_base(const lvsr_model* m, int l, int dir) {
  char buf[128];
  if (encoder_dirs(m) == 1)
    snprintf(buf, sizeof(buf), "/recognizer/encoder/with_fork%d", l);
  else
    snprintf(buf, sizeof(buf), "/recognizer/encoder/bidir%d/%s", l, dir ? "backward" : "forward");
  return buf;
}

static inline PriorParams prior_of(const lvsr_config& c) {
  PriorParams p;
  p.type = c.prior_type;
  p.initial_begin = c.prior_initial_begin;
  p.initial_end = c.prior_initial_end;
  p.min_speed = c.prior_min_speed;
  p.max_speed = c.prior_max_speed;
  p.before = c.prior_before;
  p.after = c.prior_after;
  return p;
}

// Host calls without a stream take effect after all work queued on the handle: they copy on its bound stream and,
// when the copy touches host memory, wait for it.
static inline int copy_on_handle(const lvsr_model* m, void* dst, const void* src, size_t bytes, cudaMemcpyKind kind) {
  LVSR_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, kind, m->stream));
  LVSR_CUDA_OK(cudaStreamSynchronize(m->stream));
  return 0;
}

struct ArenaScope {
  Arena& ws;
  cudaStream_t st;
  ArenaScope(lvsr_model* mm, cudaStream_t s) : ws(mm->ws), st(s) { ws.enter(); }
  ArenaScope(Arena& a, cudaStream_t s) : ws(a), st(s) { ws.enter(); }
  ~ArenaScope() { ws.leave(st); }
};

// Rewinds the workspace to its construction-time offset when the scope ends, unless it overflowed (off > cap)
struct ArenaMark { Arena& ws; const size_t off = ws.off; ~ArenaMark() { if (ws.off <= ws.cap) ws.off = off; } };

// Features encoder layer 0 takes: the bottom MLP's last width, or the recordings' features without one
static inline int encoder_input_dim(const lvsr_model* m) {
  return m->bottom.num_layers ? m->bottom.dims[m->bottom.num_layers - 1] : m->cfg.num_features;
}
// Bottom layer i: its Blocks path (MLP "bottom" of the brick "bottom", linears "linear_<i>") and input width
static inline std::string bottom_linear(int i) { return "/recognizer/bottom/bottom/linear_" + std::to_string(i); }
static inline int bottom_input_dim(const lvsr_model* m, int i) { return i ? m->bottom.dims[i - 1] : m->cfg.num_features; }

// A packed fork, blocks in column order: <fork>/<param>.W fills columns [col, col + cols) of W [rows, ld], .b those of b [ld]
struct ForkLayout { std::string fork; int rows, ld; struct { std::string param; int col, cols; } block[2]; };
// encoder layer l, direction dir, in Wcat[l] / bcat[l]: per direction [inputs D | gate_inputs 2D (update | reset)],
// encoder_dirs(m) directions side by side
static inline ForkLayout encoder_fork(const lvsr_model* m, int l, int dir) {
  const lvsr_config& c = m->cfg;
  const int D = c.dims_bidir[l], c0 = dir * 3 * D, din = l ? encoder_output_dim(m, l - 1) : encoder_input_dim(m);
  return {enc_base(m, l, dir) + "/fork", din, 3 * encoder_dirs(m) * D,
          {{"fork_inputs", c0, D}, {"fork_gate_inputs", c0 + D, 2 * D}}};
}
// Suffix of the names of decoder layer l's inputs: "" for layer 0, "#<l>" above it (the RecurrentStack's names of
// layer l's sequences, libs/blocks/blocks/bricks/recurrent.py:819-820)
static inline std::string layer_suffix(int l) { return l ? "#" + std::to_string(l) : ""; }
// fork(feedback(y)) of decoder layer l in dec[l].Wff / dec[l].bff: [gate_inputs 2C | inputs C]
static inline ForkLayout feedback_fork(const lvsr_config& c, int l) {
  const std::string x = layer_suffix(l);
  return {std::string(GEN) + "/fork", c.dim_feedback, 3 * c.dim_dec,
          {{"fork_gate_inputs" + x, 0, 2 * c.dim_dec}, {"fork_inputs" + x, 2 * c.dim_dec, c.dim_dec}}};
}

static inline int check_ready(lvsr_model* m) {
  LVSR_CHECK(m != nullptr, "null model");
  if (!m->finalized) {
    if (m->noise.stale) {             // the update may still run on its own stream: pack the means once it is done
      LVSR_CUDA_OK(cudaDeviceSynchronize());
      m->noise.stale = false;
    }
    return lvsr_model_finalize(m);
  }
  return 0;
}

// One encoder layer as the training step's backward pass reads it.
struct LayerTape {
  const float* X;      // input of the layer [T*B, Din]
  float* pre;          // [T*B, 3 ndir D] forward tape, then dPre
  float* hext;         // [(T+2), B, ndir D]
  int T, Din, D, k;
  long long mstride;
};

// shared orchestration pieces (api.cu)
int finalize_on_stream(lvsr_model* m, cudaStream_t st, bool synchronise);
int copy2d(float* dst, int ld_dst, const float* src, int ld_src, int rows, int cols, cudaStream_t st);   // float matrices
// a packed fork's blocks, W first: parameters -> W / b (grads null), or W / b (gradients) -> the flat gradient buffer
int fork_copy(lvsr_model* m, const ForkLayout& f, float* W, float* b, float* grads, cudaStream_t st);
// adaptive weight noise (noise.cu): the sample pass of a training forward (noisy parameters + priors + model cost)
// and the gradient transform of an update (both gradient groups; *nparts partial sums of squares of their union in
// noise.norm_part when nparts is not null).
int noise_sample(lvsr_model* m, cudaStream_t st);
int noise_gradients(lvsr_model* m, float* grads, float gscale, float* gls2, cudaStream_t st, int* nparts);
// dropout and weight noise (noise.cu): out = in * the dropout multiplier of update `update` over a [T, B, F] batch whose
// first utterance has the global index utt_offset (in null: the multiplier itself; in == out is allowed), and the
// noisy parameter copy reg.noisy of the handle's current update.
struct DropoutKey { unsigned long long seed; long long update, utt_offset; };
int dropout_apply(const DropoutKey& key, const float* in, float* out, int T, int B, int F, cudaStream_t st);
int weight_noise_sample(lvsr_model* m, cudaStream_t st);
// Every encoder layer (fork projection + BiGRU scan) and the mask of the encoded frames: attended [Tp, B, E] (the last
// layer writes it), attended_mask [Tp, B].  Buffers come from `ws`.  Without a tape (inference) the BiGRU runs without
// the training stores; with one, tape[l] records layer l's buffers (and allocates hext) for the backward pass.
// With a bottom MLP it runs first, on all T*B frames; with a tape, bottom_out[i] (LVSR_MAX_BOTTOM entries) records
// the output of its layer i, after the activation, for the backward pass.  dropout (null: none) multiplies the input of
// layer 0 by its mask, in a copy from `ws` that layer 0's tape records; bottom_out keeps the undropped outputs.
int run_encoder(lvsr_model* m, Arena& ws, const float* x, const float* mask, int T, int B, float* attended,
                float* attended_mask, LayerTape* tape, cudaStream_t st, const float** bottom_out = nullptr,
                const DropoutKey* dropout = nullptr);
// The bottom MLP (bottom.cu): out[i] = act(X_i W_i + b_i) for every layer over `rows` frames, buffers from `ws`
int bottom_forward(lvsr_model* m, Arena& ws, const float* x, int rows, const float** out, cudaStream_t st);
// dY [rows, n] <- dY * act'(Y) in place, from the layer's output Y = act(pre) (bottom.cu)
int bottom_act_backward(float* dY, const float* Y, long long n, int activation, cudaStream_t st);
size_t bottom_ws_bytes(const lvsr_model* m, int rows);
// out[M, N] = A[M, K] . W + bias on the tensor cores when tw holds a packed form and the shape suits it, else on FFMA
// tiles; *kpad (may be null) = the contraction as the tensor-core GEMM stored it, 0 on FFMA; *operands (may be null) =
// LVSR_ENC_OPS_* of the kernel that ran
int projection_gemm(Arena& ws, const float* A, int M, int K, const float* W, const TcWeights* tw, int N,
                    const float* bias, float* out, cudaStream_t st, int* kpad = nullptr, int* operands = nullptr);
// Readout.merge of R step-wise rows into merged [R, post_merge_dim], then the post-merge body: *tail = the input of
// the readout tail (readout_args).  Depth 1: merged itself; deeper: merged holds h_0 = act(merge + post_merge/bias.b)
// and the body runs on buffers from m->ws.
int readout_merged(lvsr_model* m, int R, const float* states, const float* ctx, float* merged, const float** tail,
                   cudaStream_t st);
// The post-merge body above h_0 [R, d_1] at depth k > 1: h_j = act(h_{j-1} W_{j-1} + b_{j-1}) for j = 1 .. k-2 (the bias
// and the activation in the product's epilogue) and *tail = z = h_{k-2} W_{k-2}, whose bias and activation the tail
// applies.  bulk: the tile GEMM (L*B teacher-forced rows), else dense_step.  Buffers from ws; hidden (null: not kept)
// receives h_0 .. h_{k-2}.  Depth 1: *tail = h0, nothing runs.
int readout_body(lvsr_model* m, Arena& ws, int R, const float* h0, bool bulk, const float** tail, const float** hidden,
                 cudaStream_t st);
// The readout tail (readout_costs) on `tail`: bias + activation + the last Linear + emitter.  Depth 1: post_merge/bias.b
// and linear_0; deeper: linear_{k-2}.b and linear_{k-1}.
ReadoutArgs readout_args(lvsr_model* m, int R, const float* tail);
// language model (api.cu): the device view of the attached FST, the fusion fields of a readout, and the LM status
// word read back after a synchronisation of st (an error return when a kernel reported one; the word is cleared)
static inline bool lm_attached(const lvsr_model* m) { return (bool)m->lm_off; }
// task loss estimation (lvsr_model_set_criterion): RewardRegressionEmitter instead of SoftmaxEmitter
static inline bool tle_criterion(const lvsr_model* m) { return m->criterion.name != LVSR_CRITERION_LOG_LIKELIHOOD; }
// the emitter's initial output: num_phonemes for SoftmaxEmitter (lvsr/bricks/recognizer.py:286), the criterion's for
// RewardRegressionEmitter (0 in the reference, lvsr/bricks/__init__.py:198-201)
static inline int initial_output(const lvsr_model* m) {
  return tle_criterion(m) ? m->criterion.initial_output : m->cfg.num_phonemes;
}
LmFst lm_fst(lvsr_model* m);
void lm_fuse(const lvsr_model* m, ReadoutArgs& r, const float* lm_add);
int lm_report(unsigned status);
size_t encoder_ws_bytes(const lvsr_model* m, int T, int B);
size_t cost_ws_bytes(const lvsr_model* m, int Tp, int B, int L);
// lvsr_cost_matrix_groundtruth, which under a task-loss criterion keeps what the loss was formed from in `tle` (null:
// workspace scratch): the emitter costs (-readouts), rewards and gains, each [L*B, num_phonemes].  With `tle` given the
// call does not wait for the groundtruth's eos check: the caller runs tle_check_status once its own work is enqueued.
struct TleTape { float *neg, *rewards, *gains; };
// Synchronises st, then reports the first utterance of the last reward launch whose groundtruth holds no eos
int tle_check_status(lvsr_model* m, cudaStream_t st);
int cost_matrix(lvsr_model* m, const float* attended, const float* attended_mask, int Tp, int B, const int64_t* labels,
                const float* labels_mask, int L, const int64_t* groundtruth, int Lg, float* costs, float* weights_out,
                float* energies_out, float* states_out, float* wavg_out, const TleTape* tle, cudaStream_t st);
// generate() under RewardRegressionEmitter for n steps on the device (glimpses, readout, arg-max, transition per step,
// no host round trip): prediction [n, B] and its mask [n, B] (1 up to and including the first eos), as
// lvsr/main.py:245-283 builds them for greedy exploration.  Buffers from m->ws.
int tle_generate_greedy(lvsr_model* m, const float* attended, const float* attended_mask, int Tp, int B, int n,
                        long long* prediction, float* prediction_mask, cudaStream_t st);

// The two device steps of lvsr_beam_search_many (search.cu), which holds the device guard and has finalized the
// model.  The hypotheses (rows) of utterance s are the contiguous rows [seg_start[s], seg_start[s+1]) -- one segment
// is what the reference calls the batch inside BeamSearch.search, so the batch-global window cut of take_glimpses
// is taken per segment.  row_utt[r] = column of the row's utterance in attended / preprocessed / attended_mask
// [T',U,.]; row_seg[r] = its segment; utt_len[s] = valid encoded frames of the segment's utterance.
//
// search_expand = logprobs_computer + BeamSearch._smallest (B/search.py:109-117,220-242,341-344): take_glimpses once
// per row (kept in wavg / new_weights / new_energies for search_advance), readout, -log softmax, and per segment the
// k smallest cost_so_far + (-logp) in increasing order: top_parent (row index), top_symbol, top_cost [nseg * k],
// top_count [nseg] (= min(k, width * V); -1 if a log-probability was not finite).
// lm_add [R, V] (null without a language model) is fused into the readout.
int search_expand(lvsr_model* m, const float* attended, const float* preprocessed, const float* attended_mask, int Tp,
                  int U, const int* utt_len, const int* row_utt, const int* row_seg, const int* seg_start, int nseg,
                  int R, const float* states, const float* weights, const long long* step, const float* cost_so_far,
                  const float* lm_add, int k, float* wavg, float* new_weights, float* new_energies, int* top_parent,
                  int* top_symbol, float* top_cost, int* top_count, cudaStream_t st);
// search_advance = next_state_computer (B/search.py:119-142) for the Rn selected children (parent rows + symbols):
// gathers the parents' state and, under the expanding prior and for content attention, their glimpses from
// search_expand (exact there because the window does not depend on which rows are in the batch); under the
// window_around_* priors it recomputes
// take_glimpses over the selected rows as the reference does.  Then Distribute + GRU step; step + 1.
int search_advance(lvsr_model* m, const float* attended, const float* preprocessed, const float* attended_mask, int Tp,
                   int U, const int* utt_len, int Rn, const int* parent, const long long* symbols, const int* row_utt,
                   const int* row_seg, const int* seg_start, int nseg, const float* states, const float* weights,
                   const long long* step, const float* wavg, const float* new_weights, const float* new_energies,
                   float* n_states, float* n_wavg, float* n_weights, float* n_energies, long long* n_step,
                   cudaStream_t st);

}  // namespace lvsr
