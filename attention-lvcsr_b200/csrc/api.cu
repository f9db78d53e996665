// C ABI of the H100-native attention-lvcsr hot path (see include/lvsr_b200.h).
//
// Host-side orchestration only: which kernel runs when, on which buffers.  The
// compiled-function seam it replaces is SURVEY.md section 8b tier b3
// (libs/blocks/blocks/search.py:97-142; lvsr/bricks/recognizer.py:375-390,490-494).
// The persistent decoder's hand-over buffers, their sentinel pre-fill, its plan and its debug switches are
// dec_scan.cu's (run_dec_scan); lvsr_cost_matrix only chooses between it and the step-wise kernels.
#include "lvsr_b200.h"

#include <stdarg.h>
#include <stdlib.h>

#include <algorithm>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "model.h"

namespace lvsr {

thread_local std::string g_last_error;
long long g_launch_count = 0;
std::atomic<long long> g_device_bytes{0};

int set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return 1;
}

// ---- per-kernel-class event timing ---------------------------------------------------
struct ProfEntry { std::string cls; cudaEvent_t a, b; };
static bool g_prof_on = false;
static std::vector<ProfEntry> g_prof;

ProfScope::ProfScope(const char* kernel_class, cudaStream_t stream) : slot(-1), st(stream) {
  if (!g_prof_on) return;
  ProfEntry e;
  e.cls = kernel_class;
  if (cudaEventCreate(&e.a) != cudaSuccess || cudaEventCreate(&e.b) != cudaSuccess) return;
  cudaEventRecord(e.a, st);
  g_prof.push_back(e);
  slot = (int)g_prof.size() - 1;
}
ProfScope::~ProfScope() {
  if (slot >= 0) cudaEventRecord(g_prof[slot].b, st);
}

}  // namespace lvsr

using namespace lvsr;

namespace lvsr {

void add_param(lvsr_model* m, const std::string& name, int64_t d0, int64_t d1 = -1) {
  Param p;
  p.name = name;
  p.shape[0] = d0;
  p.shape[1] = d1 > 0 ? d1 : 1;
  p.ndim = d1 > 0 ? 2 : 1;
  p.count = d0 * (d1 > 0 ? d1 : 1);
  p.dev = nullptr;
  m->index[name] = (int)m->params.size();
  m->params.push_back(p);
}


// Blocks initialisation order (oracle/lvsr_oracle.py: param_shapes)
void build_param_table(lvsr_model* m) {
  const lvsr_config& c = m->cfg;
  int din = encoder_input_dim(m);
  for (int l = 0; l < c.num_layers; ++l) {
    const int D = c.dims_bidir[l];
    for (int dir = 0; dir < encoder_dirs(m); ++dir) {
      const std::string b = enc_base(m, l, dir);
      add_param(m, b + "/gatedrecurrent.state_to_state", D, D);
      add_param(m, b + "/gatedrecurrent.state_to_gates", D, 2 * D);
      add_param(m, b + "/gatedrecurrent.initial_state", D);
      add_param(m, b + "/fork/fork_inputs.b", D);
      add_param(m, b + "/fork/fork_inputs.W", din, D);
      add_param(m, b + "/fork/fork_gate_inputs.b", 2 * D);
      add_param(m, b + "/fork/fork_gate_inputs.W", din, 2 * D);
    }
    din = encoder_output_dim(m, l);
  }
  // SpeechRecognizer.children = [encoder, top, bottom, generator] (lvsr/bricks/recognizer.py:350); Linear._allocate
  // makes W before b (libs/blocks/blocks/bricks/simple.py)
  for (int i = 0; i < m->bottom.num_layers; ++i) {
    add_param(m, bottom_linear(i) + ".W", bottom_input_dim(m, i), m->bottom.dims[i]);
    add_param(m, bottom_linear(i) + ".b", m->bottom.dims[i]);
  }
  const int E = m->E, C = c.dim_dec, M = c.dim_matcher, K = c.conv_num_filters, w = 2 * c.conv_n + 1;
  const int V = c.num_phonemes, Cfb = c.dim_feedback, Cpm = c.post_merge_dim;
  const std::string g = GEN, t = TR, a = att_base(m);
  // dec_stack 2: every consumer of the states takes one more input, "states#1", and every consumer of the
  // transition's sequences "inputs#1" / "gate_inputs#1" (the RecurrentStack's names for layer 1, recurrent.py:819-820)
  const bool stack = c.dec_stack == 2;
  if (!c.one_of_n_feedback) add_param(m, g + "/readout/lookupfeedback/lookuptable.W", V + 1, Cfb);
  if (c.use_states_for_readout) {
    add_param(m, g + "/readout/merge/transform_states.W", C, Cpm);
    if (stack) add_param(m, g + "/readout/merge/transform_states#1.W", C, Cpm);
  }
  add_param(m, g + "/readout/merge/transform_weighted_averages.W", E, Cpm);
  add_param(m, g + "/readout/post_merge/bias.b", Cpm);
  // MLP.children = [linear_0 .. linear_{k-1}]; Linear._initialize draws b before W (B/bricks/interfaces.py:195-200)
  for (int j = 0, k = readout_depth(m); j < k; ++j) {
    const int din = j ? readout_dim(m, j) : Cpm / c.maxout_pieces, dout = j + 1 < k ? readout_dim(m, j + 1) : V;
    add_param(m, readout_linear(j) + ".b", dout);
    add_param(m, readout_linear(j) + ".W", din, dout);
  }
  add_param(m, g + "/fork/fork_inputs.b", C);
  add_param(m, g + "/fork/fork_inputs.W", Cfb, C);
  add_param(m, g + "/fork/fork_gate_inputs.b", 2 * C);
  add_param(m, g + "/fork/fork_gate_inputs.W", Cfb, 2 * C);
  if (stack) {
    add_param(m, g + "/fork/fork_inputs#1.b", C);
    add_param(m, g + "/fork/fork_inputs#1.W", Cfb, C);
    add_param(m, g + "/fork/fork_gate_inputs#1.b", 2 * C);
    add_param(m, g + "/fork/fork_gate_inputs#1.W", Cfb, 2 * C);
  }
  // AttentionRecurrent.children = [transition, attention, distribute]; RecurrentStack.children = transitions + forks,
  // and fork_1 (outputs: layer 1's own sequence names) has no bias under skip_connections (recurrent.py:818-831)
  for (int l = 0; l < c.dec_stack; ++l) {
    add_param(m, dec_gru(m, l) + ".state_to_state", C, C);
    add_param(m, dec_gru(m, l) + ".state_to_gates", C, 2 * C);
    add_param(m, dec_gru(m, l) + ".initial_state", C);
  }
  if (stack) {
    add_param(m, t + "/recurrentstack/fork_1/fork_inputs.W", C, C);
    add_param(m, t + "/recurrentstack/fork_1/fork_gate_inputs.W", C, 2 * C);
  }
  add_param(m, a + "/state_trans/transform_states.W", C, M);
  if (stack) add_param(m, a + "/state_trans/transform_states#1.W", C, M);
  add_param(m, a + "/preprocess.b", M);
  add_param(m, a + "/preprocess.W", E, M);
  if (c.energy_normalizer != LVSR_NORM_SOFTMAX) add_param(m, a + "/energy_comp/linear.b", 1);
  add_param(m, a + "/energy_comp/linear.W", M, 1);
  if (!content_attention(m)) {            // SequenceContentAttention has no location term (B/bricks/attention.py:259-414)
    add_param(m, a + "/handler.W", K, M);
    add_param(m, a + "/conv1d.filters", K, w);
  }
  add_param(m, t + "/distribute/fork_inputs.W", E, C);
  add_param(m, t + "/distribute/fork_gate_inputs.W", E, 2 * C);
  if (stack) {
    add_param(m, t + "/distribute/fork_inputs#1.W", E, C);
    add_param(m, t + "/distribute/fork_gate_inputs#1.W", E, 2 * C);
  }
}

int copy2d(float* dst, int ld_dst, const float* src, int ld_src, int rows, int cols, cudaStream_t st) {
  LVSR_CUDA_OK(cudaMemcpy2DAsync(dst, (size_t)ld_dst * sizeof(float), src, (size_t)ld_src * sizeof(float),
                                 (size_t)cols * sizeof(float), rows, cudaMemcpyDeviceToDevice, st));
  return 0;
}

int fork_copy(lvsr_model* m, const ForkLayout& f, float* W, float* b, float* grads, cudaStream_t st) {
  for (int bias = 0; bias < 2; ++bias)
    for (const auto& k : f.block) {
      const Param* p = m->param(f.fork + "/" + k.param + (bias ? ".b" : ".W"));
      LVSR_CHECK(p, "fork_copy: %s has no parameter %s", f.fork.c_str(), k.param.c_str());
      float* packed = (bias ? b : W) + k.col;
      if (int rc = grads ? copy2d(grads + p->offset, k.cols, packed, f.ld, bias ? 1 : f.rows, k.cols, st)   // scatter gradients
                         : copy2d(packed, f.ld, p->dev, k.cols, bias ? 1 : f.rows, k.cols, st)) return rc;   // pack parameters
    }
  return 0;
}

// The weights that map a decoder state row to the attention's match space and to the readout's merge.  With
// dec_stack 2 the state is [s0 | s1] and both bricks sum one Linear per state (lvsr/bricks/attention.py:103-104,
// Merge of lvsr/bricks/recognizer.py:298-301): one product with the row-stacked weights finalize packs.
static const float* att_state_weights(const lvsr_model* m) {
  return m->cfg.dec_stack == 2 ? m->stack.Ws : m->P(att_base(m) + "/state_trans/transform_states.W");
}
static const float* readout_state_weights(const lvsr_model* m) {
  return m->cfg.dec_stack == 2 ? m->stack.Wm : m->P(std::string(GEN) + "/readout/merge/transform_states.W");
}
static const float* initial_state_row(const lvsr_model* m) {
  return m->cfg.dec_stack == 2 ? m->stack.h0 : m->P(dec_gru(m, 0) + ".initial_state");
}

// take_glimpses for R rows: q = s.W_state, window, attention step.
struct Segments {           // batched beam search: hypotheses of one utterance = one segment (the reference's batch)
  const int* seg_start = nullptr; int nseg = 0; const int* seg_len = nullptr; const int* row_seg = nullptr;
};
int glimpses(lvsr_model* m, const float* H, const float* P, const float* maskH, int Tp, int U,
             const int* row_utt, int R, const float* states, const float* w_prev, const long long* step,
             long long step_offset, float* w_out, float* e_out, float* ctx, cudaStream_t st, Segments sg = Segments()) {
  const lvsr_config& c = m->cfg;
  Arena& ws = m->ws;
  float* q = ws.f32((size_t)R * c.dim_matcher);
  int* win = ws.i32((size_t)2 * std::max(1, sg.nseg));
  float* lohi = ws.f32((size_t)2 * R);
  LVSR_CHECK(q && win && lohi, "out of device memory (workspace)");
  DenseArgs d = {};
  d.op[0] = {states, state_dim(m), state_dim(m), att_state_weights(m), c.dim_matcher};
  d.R = R; d.N = c.dim_matcher; d.mode = DENSE_PLAIN; d.out = q;
  if (int rc = dense_step(d, st)) return rc;
  WindowArgs wa = {};
  wa.weights = w_prev; wa.step = step; wa.step_offset = step_offset; wa.R = R; wa.Tp = Tp;
  wa.prior = prior_of(c); wa.win = win; wa.lohi = lohi;
  wa.seg_start = sg.seg_start; wa.nseg = sg.nseg; wa.seg_len = sg.seg_len;
  if (int rc = attention_window(wa, st)) return rc;
  AttStepArgs a = {};
  a.P = P; a.H = H; a.maskH = maskH; a.row_utt = row_utt; a.q = q; a.w_prev = w_prev; a.win = win; a.lohi = lohi;
  a.row_seg = sg.seg_start ? sg.row_seg : nullptr;
  a.filt = m->P(att_base(m) + "/conv1d.filters");     // null for content attention
  a.Wh = m->P(att_base(m) + "/handler.W");
  a.v = m->P(att_base(m) + "/energy_comp/linear.W");
  a.v_bias = m->v_bias;   // energy bias exists only when the normaliser is not softmax
  a.w_out = w_out; a.e_out = e_out; a.ctx = ctx;
  a.R = R; a.U = U; a.Tp = Tp; a.M = c.dim_matcher; a.E = m->E; a.K = c.conv_num_filters; a.n = c.conv_n;
  a.normalizer = c.energy_normalizer;
  return attention_step(a, !content_attention(m), &m->att_cs, st);
}

// compute_states for R state rows of stride S = state_dim(m): distribute + fork(feedback) + GRU step, layer by layer.
// Layer l reads states[:, lC : (l+1)C] and writes next_states[:, lC : (l+1)C]; with dec_stack 2, layer 1 also takes
// layer 0's new state next_states[:, :C] through the RecurrentStack's bias-free fork_1 (recurrent.py:925-950).  The
// layers share one z / hr / ai scratch set (stream order).  next_states may be states: each launch reads a state
// element before the launch that overwrites it, or in the thread that overwrites it.
static int transition(lvsr_model* m, int R, const float* states, const float* ctx, const long long* outputs,
                      const float* rmask, float* next_states, cudaStream_t st) {
  const lvsr_config& c = m->cfg;
  Arena& ws = m->ws;
  const int C = c.dim_dec, S = state_dim(m);
  float* z = ws.f32((size_t)R * C);
  float* hr = ws.f32((size_t)R * C);
  float* ai = ws.f32((size_t)R * C);
  LVSR_CHECK(z && hr && ai, "out of device memory (workspace)");
  for (int l = 0; l < c.dec_stack; ++l) {
    const lvsr_model::DecLayer& in = m->dec[l];
    const float* s = states + (size_t)l * C;
    DenseArgs g = {};
    g.op[0] = {ctx, m->E, m->E, in.Wd.get(), 3 * C};
    if (l == 1) g.op[1] = {next_states, C, S, m->stack.F, 3 * C};
    g.op[l + 1] = {s, C, S, m->P(dec_gru(m, l) + ".state_to_gates"), 2 * C};   // the layer's own state comes last
    g.add = in.FF.get(); g.arow = outputs; g.add_rows = c.num_phonemes + 1; g.R = R; g.N = 3 * C; g.mode = DENSE_GATES;
    g.s = s; g.ld_s = S; g.z = z; g.hr = hr; g.ai = ai; g.C = C;
    if (int rc = dense_step(g, st)) return rc;
    DenseArgs k = {};
    k.op[0] = {hr, C, C, m->P(dec_gru(m, l) + ".state_to_state"), C};
    k.add = ai; k.arow = nullptr; k.R = R; k.N = C; k.mode = DENSE_CAND;
    k.s = s; k.ld_s = S; k.z = z; k.rmask = rmask; k.out = next_states + (size_t)l * C; k.ld_out = S; k.C = C;
    if (int rc = dense_step(k, st)) return rc;
  }
  return 0;
}

int readout_merged(lvsr_model* m, int R, const float* states, const float* ctx, float* merged, const float** tail,
                   cudaStream_t st) {
  const lvsr_config& c = m->cfg;
  const bool deep = readout_depth(m) > 1;
  DenseArgs d = {};
  const int S = state_dim(m), N = c.post_merge_dim;
  d.op[0] = {ctx, m->E, m->E, m->P(std::string(GEN) + "/readout/merge/transform_weighted_averages.W"), N};
  if (c.use_states_for_readout) d.op[1] = {states, S, S, readout_state_weights(m), N};
  d.R = R; d.N = N; d.mode = DENSE_PLAIN; d.out = merged;
  if (deep) {                      // h_0 = act(merge + post_merge/bias.b) in the merge's epilogue
    d.mode = DENSE_ACT;
    d.bias = m->P(std::string(GEN) + "/readout/post_merge/bias.b");
    d.act = c.post_merge_activation;
  }
  if (int rc = dense_step(d, st)) return rc;
  return readout_body(m, m->ws, R, merged, false, tail, nullptr, st);
}

int readout_body(lvsr_model* m, Arena& ws, int R, const float* h0, bool bulk, const float** tail, const float** hidden,
                 cudaStream_t st) {
  const int k = readout_depth(m);
  *tail = h0;
  if (k == 1) return 0;
  ProfScope prof("readout_body", st);
  const int act = m->cfg.post_merge_activation;
  const float* h = h0;
  if (hidden) hidden[0] = h0;
  for (int j = 0; j + 1 < k; ++j) {
    const int din = readout_dim(m, j), dout = readout_dim(m, j + 1);
    const bool last = j + 2 == k;
    float* out = ws.f32((size_t)R * dout);
    LVSR_CHECK(out, "out of device memory (readout hidden layer)");
    const float* W = m->P(readout_linear(j) + ".W");
    const float* b = m->P(readout_linear(j) + ".b");
    if (bulk) {
      GemmArgs g = make_gemm(h, R, din, W, dout, last ? nullptr : b, out);
      if (!last) g.act = act;
      if (int rc = gemm_bias(g, st)) return rc;
    } else {
      DenseArgs d = {};
      d.op[0] = {h, din, din, W, dout};
      d.R = R; d.N = dout; d.out = out; d.mode = last ? DENSE_PLAIN : DENSE_ACT; d.bias = b; d.act = act;
      if (int rc = dense_step(d, st)) return rc;
    }
    if (last) {
      *tail = out;
    } else {
      h = out;
      if (hidden) hidden[j + 1] = out;
    }
  }
  return 0;
}

ReadoutArgs readout_args(lvsr_model* m, int R, const float* tail) {
  const lvsr_config& c = m->cfg;
  const int k = readout_depth(m);
  ReadoutArgs r = {};
  r.merged = tail;
  r.b_pm = m->P(k == 1 ? std::string(GEN) + "/readout/post_merge/bias.b" : readout_linear(k - 2) + ".b");
  r.Wo = m->P(readout_linear(k - 1) + ".W");
  r.bo = m->P(readout_linear(k - 1) + ".b");
  r.R = R; r.Cpm = readout_dim(m, k - 1); r.pieces = c.maxout_pieces; r.V = c.num_phonemes; r.act = c.post_merge_activation;
  r.tle = tle_criterion(m) ? 1 : 0;
  return r;
}

LmFst lm_fst(lvsr_model* m) {
  LmFst f = {};
  f.off = m->lm_off.get(); f.label = m->lm_label.get(); f.next = m->lm_next.get(); f.weight = m->lm_weight.get();
  f.start = m->lm_start; f.V = m->cfg.num_phonemes;
  f.no_transition_cost = (float)m->lm_fusion.no_transition_cost;
  f.status = m->lm_status.get();
  return f;
}

void lm_fuse(const lvsr_model* m, ReadoutArgs& r, const float* lm_add) {
  const lvsr_lm_fusion& u = m->lm_fusion;
  r.lm_add = lm_add;
  r.lm_weight = (float)u.weight; r.am_beta = (float)u.am_beta;
  r.norm_am = u.normalize_am_weights != 0; r.norm_lm = u.normalize_lm_weights != 0;
  r.norm_tot = u.normalize_tot_weights != 0;
}

int lm_report(unsigned status) {
  LVSR_CHECK(status != LVSR_LM_TOO_MANY_STATES, "language model: a hypothesis reached more than %d FST states",
             (int)LVSR_LM_MAX_STATES);
  LVSR_CHECK(status != LVSR_LM_CLOSURE_CAP, "language model: an epsilon closure exceeded 32 FST states");
  LVSR_CHECK(status != LVSR_LM_CYCLE, "language model: the FST has an epsilon cycle");
  LVSR_CHECK(status == 0, "language model: status %u", status);
  return 0;
}

// Synchronises st and turns the LM status word into an error return (clearing it).
static int lm_sync_status(lvsr_model* m, cudaStream_t st) {
  unsigned h = 0;
  LVSR_CUDA_OK(cudaMemcpyAsync(&h, m->lm_status.get(), sizeof(h), cudaMemcpyDeviceToHost, st));
  LVSR_CUDA_OK(cudaStreamSynchronize(st));
  if (h) LVSR_CUDA_OK(cudaMemsetAsync(m->lm_status.get(), 0, sizeof(unsigned), st));
  return lm_report(h);
}

size_t encoder_ws_bytes(const lvsr_model* m, int T, int B) {
  size_t total = 0;
  int Tl = T;
  for (int l = 0; l < m->cfg.num_layers; ++l) {
    const int D = m->cfg.dims_bidir[l], k = m->cfg.subsample[l], nd = encoder_dirs(m);
    const int Tout = ceil_div(Tl, k);
    total += ((size_t)Tl * B * 3 * nd * D + (size_t)Tout * B * nd * D) * sizeof(float) + 1024;
    total += (size_t)2 * Tl * B * gemm_tc_kpad(l == 0 ? encoder_input_dim(m) : encoder_output_dim(m, l - 1)) * sizeof(float) + 1024;
    total += gemm_f16_stream_sync_ints(Tl * B) * sizeof(int) + 1024;   // scheduling area of a streamed projection
    Tl = Tout;
  }
  return total + bottom_ws_bytes(m, T * B) + (1 << 16);
}
size_t cost_ws_bytes(const lvsr_model* m, int Tp, int B, int L) {
  const lvsr_config& c = m->cfg;
  const size_t S = state_dim(m);
  size_t f = (size_t)Tp * B * c.dim_matcher + (size_t)2 * Tp * B * m->E + (size_t)(L + 1) * B * S + (size_t)L * B * m->E +
             (size_t)4 * B * Tp + (size_t)L * B * c.post_merge_dim + (size_t)B * c.dim_matcher +
             (size_t)L * B * (Tp + c.dim_matcher + S + 1) +
             (size_t)3 * B * c.dim_dec + 4 * B + 64 + (size_t)L * B * readout_hidden_floats(m);
  return f * sizeof(float) + (1 << 16);
}



}  // namespace lvsr

extern "C" {

const char* lvsr_last_error(void) { return g_last_error.c_str(); }
int lvsr_version(void) { return 104; }
int64_t lvsr_launch_count(int reset) {
  const int64_t v = g_launch_count;
  if (reset) g_launch_count = 0;
  return v;
}
int64_t lvsr_device_bytes(void) { return g_device_bytes.load(); }

int lvsr_profile_enable(int on) {
  g_prof_on = on != 0;
  return 0;
}
int lvsr_profile_read(const char* kernel_class, double* total_ms, int64_t* count) {
  LVSR_CHECK(kernel_class && total_ms && count, "null argument");
  LVSR_CUDA_OK(cudaDeviceSynchronize());
  double tot = 0.0;
  int64_t n = 0;
  std::vector<ProfEntry> keep;
  for (auto& e : g_prof) {
    if (e.cls == kernel_class) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, e.a, e.b) == cudaSuccess) { tot += ms; n++; }
      cudaEventDestroy(e.a);
      cudaEventDestroy(e.b);
    } else {
      keep.push_back(e);
    }
  }
  g_prof.swap(keep);
  *total_ms = tot;
  *count = n;
  return 0;
}

int lvsr_model_create(const lvsr_config* cfg, lvsr_model** out) { return lvsr_model_create_encoder(cfg, nullptr, 1, out); }

int lvsr_model_create_bottom(const lvsr_config* cfg, const lvsr_bottom_config* bottom, lvsr_model** out) {
  return lvsr_model_create_encoder(cfg, bottom, 1, out);
}

int lvsr_readout_max_width(void) {
  int H = 0;
  while (readout_smem_bytes(H + 8) <= READOUT_SMEM_LIMIT && readout_bwd_smem_bytes(H + 8) <= READOUT_SMEM_LIMIT) H += 8;
  return H;
}

int lvsr_model_create_encoder(const lvsr_config* cfg, const lvsr_bottom_config* bottom, int32_t bidir, lvsr_model** out) {
  return lvsr_model_create_readout(cfg, bottom, bidir, nullptr, out);
}

int lvsr_model_create_readout(const lvsr_config* cfg, const lvsr_bottom_config* bottom, int32_t bidir,
                              const lvsr_readout_config* readout, lvsr_model** out) {
  LVSR_CHECK(cfg && out, "null argument");
  LVSR_CHECK(bidir == 0 || bidir == 1, "bidir %d unsupported (1: bidirectional encoder, 0: forward-only encoder)", bidir);
  if (bottom) {
    LVSR_CHECK(bottom->num_layers >= 0 && bottom->num_layers <= LVSR_MAX_BOTTOM, "bottom MLP: %d layers (0 .. %d)",
               bottom->num_layers, (int)LVSR_MAX_BOTTOM);
    for (int i = 0; i < bottom->num_layers; ++i)
      LVSR_CHECK(bottom->dims[i] >= 1 && bottom->dims[i] <= LVSR_MAX_BOTTOM_DIM, "bottom MLP: width %d of layer %d (1 .. %d)",
                 bottom->dims[i], i, (int)LVSR_MAX_BOTTOM_DIM);
    LVSR_CHECK(bottom->num_layers == 0 || bottom->activation == LVSR_ACT_RELU || bottom->activation == LVSR_ACT_TANH,
               "bottom MLP: activation %d unsupported (Rectifier or Tanh)", bottom->activation);
  }
  LVSR_CHECK(cfg->num_layers >= 1 && cfg->num_layers <= LVSR_MAX_LAYERS, "num_layers %d out of range", cfg->num_layers);
  for (int l = 0; l < cfg->num_layers; ++l) {
    LVSR_CHECK(bigru_supported(cfg->dims_bidir[l]), "encoder dim %d of layer %d unsupported (a multiple of 64 from 64 to 512)",
               cfg->dims_bidir[l], l);
    LVSR_CHECK(cfg->subsample[l] >= 1, "subsample must be >= 1");
  }
  LVSR_CHECK(cfg->dim_dec % 8 == 0 && cfg->post_merge_dim % 8 == 0, "dim_dec and post_merge_dim must be multiples of 8");
  LVSR_CHECK(cfg->dim_matcher == 128 || cfg->dim_matcher == 256 || cfg->dim_matcher == 512,
             "dim_matcher %d unsupported by the attention kernel (128, 256 or 512)", cfg->dim_matcher);
  LVSR_CHECK(cfg->one_of_n_feedback ? cfg->dim_feedback == cfg->num_phonemes + 1 : cfg->dim_feedback % 4 == 0,
             "dim_feedback must be a multiple of 4 (LookupFeedback) or num_phonemes + 1 (OneOfNFeedback)");
  LVSR_CHECK(cfg->maxout_pieces >= 1 && cfg->post_merge_dim % cfg->maxout_pieces == 0, "bad maxout_pieces");
  LVSR_CHECK(cfg->post_merge_activation >= LVSR_ACT_MAXOUT && cfg->post_merge_activation <= LVSR_ACT_IDENTITY,
             "bad post_merge_activation");
  LVSR_CHECK(cfg->post_merge_activation == LVSR_ACT_MAXOUT || cfg->maxout_pieces == 1,
             "maxout_pieces must be 1 unless the activation is Maxout");
  LVSR_CHECK(cfg->attention_type == LVSR_ATT_CONTENT_AND_CONV || cfg->attention_type == LVSR_ATT_CONTENT,
             "attention_type %d unsupported (0: content_and_conv, 1: content)", cfg->attention_type);
  const bool content = cfg->attention_type == LVSR_ATT_CONTENT;
  LVSR_CHECK(content || (cfg->conv_num_filters >= 1 && cfg->conv_num_filters <= 16), "conv_num_filters %d not in [1,16]",
             cfg->conv_num_filters);
  // the centre crop [:, :, n:-n] of the reference is EMPTY for n = 0 (lvsr/bricks/attention.py:109-110)
  LVSR_CHECK(content || cfg->conv_n >= 1, "conv_n must be >= 1 (got %d)", cfg->conv_n);
  LVSR_CHECK(cfg->num_phonemes >= 1 && cfg->num_phonemes <= 128, "num_phonemes out of range");
  LVSR_CHECK(cfg->dec_stack >= 0 && cfg->dec_stack <= 2, "dec_stack %d unsupported (1 or 2)", cfg->dec_stack);
  lvsr_readout_config ro = {1, {cfg->post_merge_dim}};
  if (readout) {
    const int k = readout->num_layers;
    LVSR_CHECK(k >= 1 && k <= LVSR_MAX_READOUT, "post_merge_dims: %d layers (1 .. %d)", k, (int)LVSR_MAX_READOUT);
    LVSR_CHECK(readout->dims[0] == cfg->post_merge_dim, "post_merge_dims[0] = %d must equal post_merge_dim %d",
               readout->dims[0], cfg->post_merge_dim);
    for (int j = 1; j < k; ++j)
      LVSR_CHECK(readout->dims[j] >= 8 && readout->dims[j] % 8 == 0,
                 "post_merge_dims: width %d of layer %d must be a positive multiple of 8", readout->dims[j], j);
    LVSR_CHECK(k == 1 || cfg->post_merge_activation != LVSR_ACT_MAXOUT || cfg->maxout_pieces == 1,
               "post_merge_dims: %d layers under Maxout(%d): a Maxout of more than one piece takes one post-merge layer "
               "only (the reference's MLP takes d_j / pieces inputs that its Maxout divides again)", k,
               cfg->maxout_pieces);
    LVSR_CHECK(k == 1 || readout->dims[k - 1] <= lvsr_readout_max_width(),
               "post_merge_dims: last width %d above %d, the widest the readout kernels stage in shared memory",
               readout->dims[k - 1], lvsr_readout_max_width());
    ro = *readout;
  }
  int dev_count = 0;
  LVSR_CUDA_OK(cudaGetDeviceCount(&dev_count));
  LVSR_CHECK(dev_count > 0, "no CUDA device: the GPU path has no CPU fallback");
  std::unique_ptr<lvsr_model> m(new lvsr_model());      // deleted with every buffer it holds on a failed return
  m->cfg = *cfg;
  m->ndir = bidir ? 2 : 1;
  if (bottom && bottom->num_layers > 0) m->bottom = *bottom;
  m->readout = ro;
  if (m->cfg.dec_stack == 0) m->cfg.dec_stack = 1;     // callers that predate the field zero-fill it
  if (content) {
    // SequenceContentAttention takes none of these (lvsr/bricks/recognizer.py:261-265): softmax weights over every
    // frame, which is the expanding window [0, length) that never moves
    lvsr_config& c = m->cfg;
    c.conv_n = c.conv_num_filters = 0;
    c.energy_normalizer = LVSR_NORM_SOFTMAX;
    c.prior_type = LVSR_PRIOR_EXPANDING;
    c.prior_initial_begin = 0.0;
    c.prior_initial_end = 1e30;
    c.prior_min_speed = c.prior_max_speed = 0.0;
    c.prior_before = c.prior_after = 0.0;
  }
  LVSR_CUDA_OK(cudaGetDevice(&m->device));
  m->E = encoder_output_dim(m.get(), cfg->num_layers - 1);
  build_param_table(m.get());
  int64_t total = 0;
  for (auto& p : m->params) {
    p.offset = total;
    total += (p.count + 63) & ~(int64_t)63;
  }
  m->flat_count = total;
  {
    cudaError_t e = m->flat.alloc((size_t)total * sizeof(float));
    if (e != cudaSuccess)
      return set_error("cudaMalloc(parameters, %lld floats) failed: %s", (long long)total, cudaGetErrorString(e));
    cudaMemset(m->flat.get(), 0, (size_t)total * sizeof(float));
  }
  for (auto& p : m->params) p.dev = m->flat.get() + p.offset;
  if (m->status.alloc(64) != cudaSuccess) return set_error("cudaMalloc(status) failed");
  cudaMemset(m->status.get(), 0, 64);
  cudaDeviceSynchronize();      // the zeroed buffers are in place before a call on any stream reads them
  *out = m.release();
  return 0;
}

int lvsr_model_destroy(lvsr_model* m) {
  if (!m) return 0;
  DeviceGuard device_guard(m);
  cudaDeviceSynchronize();
  delete m;
  return 0;
}

int lvsr_model_status(lvsr_model* m, int32_t* launch_status, int64_t* stepwise_fallbacks) {
  DeviceGuard device_guard(m);
  LVSR_CHECK(m && launch_status, "null argument");
  unsigned hst = 0;
  if (int rc = copy_on_handle(m, &hst, m->status.get(), sizeof(hst), cudaMemcpyDeviceToHost)) return rc;   // after the handle's work
  *launch_status = (int32_t)hst;
  if (stepwise_fallbacks) *stepwise_fallbacks = m->dec_fallbacks;
  return 0;
}

int lvsr_model_decoder_plan(const lvsr_model* m, int32_t out[16]) {
  LVSR_CHECK(m && out, "null argument");
  for (int i = 0; i < 16; ++i) out[i] = m->dec_plan[i];
  out[LVSR_PLAN_ATT_CS] = m->att_cs;
  return 0;
}

int lvsr_model_encoder_plan(const lvsr_model* m, int32_t layer, int32_t out[16]) {
  LVSR_CHECK(m && out, "null argument");
  LVSR_CHECK(layer >= -1 && layer < m->cfg.num_layers, "encoder_plan: layer %d outside [-1, %d)", layer, m->cfg.num_layers);
  for (int i = 0; i < 16; ++i) out[i] = layer >= 0 ? m->enc_plan[layer][i] : 0;
  if (layer < 0) {
    out[LVSR_ENC_PROJ] = m->pre_plan[0];
    out[LVSR_ENC_KPAD] = m->pre_plan[1];
    out[LVSR_ENC_OPERANDS] = m->pre_plan[2];
  }
  return 0;
}

int lvsr_model_encoder_overlap(lvsr_model* m, int32_t layer, int32_t out[3]) {
  LVSR_CHECK(m && out, "null argument");
  LVSR_CHECK(layer >= 0 && layer < m->cfg.num_layers, "encoder_overlap: layer %d outside [0, %d)", layer, m->cfg.num_layers);
  DeviceGuard device_guard(m);
  out[0] = m->enc_overlap[layer];
  out[1] = out[2] = 0;
  if (out[0]) {
    int tiles[2];
    LVSR_CUDA_OK(cudaDeviceSynchronize());
    LVSR_CUDA_OK(cudaMemcpy(tiles, m->enc_tiles.get() + 2 * layer, sizeof(tiles), cudaMemcpyDeviceToHost));
    out[1] = tiles[0];
    out[2] = tiles[1];
  }
  return 0;
}

int lvsr_model_encoder_overlap_claims(lvsr_model* m, int32_t layer, int32_t* out, int64_t count) {
  LVSR_CHECK(m && out, "null argument");
  LVSR_CHECK(layer >= 1 && layer < m->cfg.num_layers && m->enc_overlap[layer],
             "encoder_overlap_claims: layer %d did not overlap in the last encoder forward", layer);
  const size_t end = layer + 1 < m->cfg.num_layers ? m->enc_claims_off[layer + 1] : m->enc_claims.bytes() / sizeof(int);
  const size_t n = end - m->enc_claims_off[layer];
  LVSR_CHECK(count >= 0 && (size_t)count <= n, "encoder_overlap_claims: %lld ints asked, layer %d has %zu",
             (long long)count, layer, n);
  DeviceGuard device_guard(m);
  LVSR_CUDA_OK(cudaDeviceSynchronize());
  LVSR_CUDA_OK(cudaMemcpy(out, m->enc_claims.get() + m->enc_claims_off[layer], (size_t)count * sizeof(int), cudaMemcpyDeviceToHost));
  return 0;
}

int lvsr_model_num_params(const lvsr_model* m) { return m ? (int)m->params.size() : 0; }
const char* lvsr_model_param_name(const lvsr_model* m, int i) {
  if (!m || i < 0 || i >= (int)m->params.size()) return nullptr;
  return m->params[i].name.c_str();
}
int lvsr_model_param_shape(const lvsr_model* m, int i, int64_t shape[2], int32_t* ndim) {
  LVSR_CHECK(m && i >= 0 && i < (int)m->params.size(), "bad parameter index %d", i);
  shape[0] = m->params[i].shape[0];
  shape[1] = m->params[i].shape[1];
  *ndim = m->params[i].ndim;
  return 0;
}
int64_t lvsr_model_flat_size(const lvsr_model* m) { return m ? m->flat_count : 0; }
int lvsr_model_param_offset(const lvsr_model* m, int i, int64_t* offset, int64_t* count) {
  LVSR_CHECK(m && offset && i >= 0 && i < (int)m->params.size(), "bad parameter index %d", i);
  *offset = m->params[i].offset;
  if (count) *count = m->params[i].count;
  return 0;
}
float* lvsr_model_flat_params(lvsr_model* m) { return m ? m->flat.get() : nullptr; }
int lvsr_model_set_param(lvsr_model* m, const char* name, const float* host, int64_t count) {
  DeviceGuard device_guard(m);
  LVSR_CHECK(m && name && host, "null argument");
  const Param* p = m->param(name);
  LVSR_CHECK(p, "unknown parameter '%s'", name);
  LVSR_CHECK(count == p->count, "parameter '%s' expects %lld values, got %lld", name, (long long)p->count, (long long)count);
  if (int rc = copy_on_handle(m, p->dev, host, (size_t)count * sizeof(float), cudaMemcpyHostToDevice)) return rc;
  m->finalized = false;
  return 0;
}
int lvsr_model_get_param(const lvsr_model* m, const char* name, float* host, int64_t count) {
  DeviceGuard device_guard(m);
  LVSR_CHECK(m && name && host, "null argument");
  const Param* p = m->param(name);
  LVSR_CHECK(p, "unknown parameter '%s'", name);
  LVSR_CHECK(count == p->count, "parameter '%s' holds %lld values, asked for %lld", name, (long long)p->count, (long long)count);
  if (int rc = copy_on_handle(m, host, p->dev, (size_t)count * sizeof(float), cudaMemcpyDeviceToHost)) return rc;
  return 0;
}

int lvsr_model_finalize(lvsr_model* m) {
  DeviceGuard device_guard(m);
  LVSR_CHECK(m, "null model");
  return finalize_on_stream(m, m->stream, true);      // after the work queued on the handle
}

int lvsr_model_clear_lm(lvsr_model* m) {
  DeviceGuard device_guard(m);
  LVSR_CHECK(m, "null model");
  if (m->lm_off) LVSR_CUDA_OK(cudaDeviceSynchronize());       // a search or cost call may still read the tables
  m->lm_off.reset(); m->lm_label.reset(); m->lm_next.reset(); m->lm_weight.reset(); m->lm_status.reset();
  return 0;
}

int lvsr_model_set_lm(lvsr_model* m, int32_t num_states, int32_t start, const int64_t* off, int64_t num_arcs,
                      const int32_t* label, const int32_t* next, const float* weight, const lvsr_lm_fusion* fusion) {
  DeviceGuard device_guard(m);
  LVSR_CHECK(m && off && fusion && num_states > 0 && num_arcs >= 0 && (num_arcs == 0 || (label && next && weight)),
             "set_lm: bad arguments");
  LVSR_CHECK(start >= 0 && start < num_states, "set_lm: start state %d outside [0, %d)", start, num_states);
  LVSR_CHECK(off[0] == 0 && off[num_states] == num_arcs, "set_lm: arc offsets must run from 0 to num_arcs");
  const int V = m->cfg.num_phonemes;
  for (int32_t s = 0; s < num_states; ++s) {
    LVSR_CHECK(off[s] <= off[s + 1], "set_lm: arc offsets decrease at state %d", s);
    for (int64_t j = off[s]; j < off[s + 1]; ++j) {
      LVSR_CHECK(label[j] >= 0 && label[j] <= V && next[j] >= 0 && next[j] < num_states,
                 "set_lm: arc %lld of state %d has label %d / next state %d out of range", (long long)j, s, label[j], next[j]);
      LVSR_CHECK(j == off[s] || label[j - 1] < label[j] || (label[j - 1] == label[j] && next[j - 1] <= next[j]),
                 "set_lm: the arcs of state %d are not sorted by (label, next state)", s);
    }
  }
  // the new tables are filled before the attached ones are replaced: a failed call leaves the handle as it was
  const size_t na = (size_t)std::max<int64_t>(num_arcs, 1);
  DeviceBuffer<unsigned> lm_status;
  DeviceBuffer<long long> lm_off;
  DeviceBuffer<int> lm_label, lm_next;
  DeviceBuffer<float> lm_weight;
  LVSR_CUDA_OK(lm_status.alloc(sizeof(unsigned)));
  LVSR_CUDA_OK(lm_off.alloc((size_t)(num_states + 1) * sizeof(long long)));
  LVSR_CUDA_OK(lm_label.alloc(na * sizeof(int)));
  LVSR_CUDA_OK(lm_next.alloc(na * sizeof(int)));
  LVSR_CUDA_OK(lm_weight.alloc(na * sizeof(float)));
  // on the handle's stream, complete before the host tables may go away
  cudaStream_t st = m->stream;
  LVSR_CUDA_OK(cudaMemsetAsync(lm_status.get(), 0, sizeof(unsigned), st));
  LVSR_CUDA_OK(cudaMemcpyAsync(lm_off.get(), off, (size_t)(num_states + 1) * sizeof(long long), cudaMemcpyHostToDevice, st));
  if (num_arcs > 0) {
    LVSR_CUDA_OK(cudaMemcpyAsync(lm_label.get(), label, (size_t)num_arcs * sizeof(int), cudaMemcpyHostToDevice, st));
    LVSR_CUDA_OK(cudaMemcpyAsync(lm_next.get(), next, (size_t)num_arcs * sizeof(int), cudaMemcpyHostToDevice, st));
    LVSR_CUDA_OK(cudaMemcpyAsync(lm_weight.get(), weight, (size_t)num_arcs * sizeof(float), cudaMemcpyHostToDevice, st));
  }
  LVSR_CUDA_OK(cudaStreamSynchronize(st));
  if (int rc = lvsr_model_clear_lm(m)) return rc;
  m->lm_status = std::move(lm_status);
  m->lm_off = std::move(lm_off);
  m->lm_label = std::move(lm_label);
  m->lm_next = std::move(lm_next);
  m->lm_weight = std::move(lm_weight);
  m->lm_start = start;
  m->lm_fusion = *fusion;
  return 0;
}

int lvsr_lm_initial_states(lvsr_model* m, int32_t R, int32_t* states, double* weights, float* add, void* stream) {
  DeviceGuard device_guard(m);
  LVSR_CHECK(m && lm_attached(m), "lm_initial_states: no language model attached");
  LVSR_CHECK(states && weights && add && R > 0, "lm_initial_states: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_stream(m, st)) return rc;
  if (int rc = lm_step(lm_fst(m), R, nullptr, nullptr, nullptr, nullptr, states, weights, add, st)) return rc;
  return lm_sync_status(m, st);
}

int lvsr_lm_next_states(lvsr_model* m, int32_t R, const int32_t* states, const double* weights, const int64_t* outputs,
                        int32_t* next_states, double* next_weights, float* next_add, void* stream) {
  DeviceGuard device_guard(m);
  LVSR_CHECK(m && lm_attached(m), "lm_next_states: no language model attached");
  LVSR_CHECK(states && weights && outputs && next_states && next_weights && next_add && R > 0,
             "lm_next_states: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_stream(m, st)) return rc;
  if (int rc = lm_step(lm_fst(m), R, states, weights, nullptr, reinterpret_cast<const long long*>(outputs), next_states,
                       next_weights, next_add, st)) return rc;
  return lm_sync_status(m, st);
}

}  // extern "C"

namespace lvsr {
// W [K, N] packed for the tensor-core GEMM into tw (allocated on first use): fp16 head/tail planes when K is a multiple
// of 64 (the forward projections' operand kind, see projection_gemm), else tf32 hi/lo planes; shapes neither kernel
// takes stay unpacked
static int pack_tc_weights(TcWeights& tw, const float* W, int K, int N, cudaStream_t st) {
  if (!tw.mem) {
    if (gemm_f16_supported(128, N, K)) {
      const size_t plane = (size_t)N * K * sizeof(__half);
      LVSR_CUDA_OK(tw.mem.alloc(2 * plane + (size_t)N * sizeof(int)));
      tw.head = reinterpret_cast<__half*>(tw.mem.get());
      tw.tail = reinterpret_cast<__half*>(tw.mem.get() + plane);
      tw.ew = reinterpret_cast<int*>(tw.mem.get() + 2 * plane);
    } else if (gemm_tc_supported(128, N, K)) {
      const size_t plane = (size_t)N * gemm_tc_kpad(K);
      LVSR_CUDA_OK(tw.mem.alloc(2 * plane * sizeof(float)));
      tw.hi = reinterpret_cast<float*>(tw.mem.get());
      tw.lo = tw.hi + plane;
    } else {
      return 0;
    }
  }
  if (tw.head) return split_weight_f16(W, K, N, tw.head, tw.tail, tw.ew, st);
  return split_weight_tf32(W, K, N, tw.hi, tw.lo, st);
}

int finalize_on_stream(lvsr_model* m, cudaStream_t st, bool synchronise) {
  const lvsr_config& c = m->cfg;
  if (m->Wcat.empty()) {       // the first finalize: the whole group, or (on a failed allocation) none of it
    std::vector<DeviceBuffer<float>> Wcat(c.num_layers), bcat(c.num_layers);
    for (int l = 0; l < c.num_layers; ++l) {
      const ForkLayout f = encoder_fork(m, l, 0);       // Wcat[l] [rows, ld], bcat[l] [ld]
      LVSR_CUDA_OK(Wcat[l].alloc((size_t)f.rows * f.ld * sizeof(float)));
      LVSR_CUDA_OK(bcat[l].alloc((size_t)f.ld * sizeof(float)));
    }
    const int C = c.dim_dec;
    lvsr_model::DecLayer dec[2];
    for (int l = 0; l < c.dec_stack; ++l) {
      lvsr_model::DecLayer& d = dec[l];
      LVSR_CUDA_OK(d.Wd.alloc((size_t)m->E * 3 * C * sizeof(float)));
      LVSR_CUDA_OK(d.Wff.alloc((size_t)c.dim_feedback * 3 * C * sizeof(float)));
      LVSR_CUDA_OK(d.bff.alloc((size_t)3 * C * sizeof(float)));
      LVSR_CUDA_OK(d.FF.alloc((size_t)(c.num_phonemes + 1) * 3 * C * sizeof(float)));
    }
    DeviceBuffer<float> Wb1;
    LVSR_CUDA_OK(Wb1.alloc((size_t)(m->E + C) * 3 * C * sizeof(float)));
    lvsr_model::Stack s;
    if (c.dec_stack == 2) {
      const size_t n[4] = {(size_t)2 * C * c.dim_matcher, (size_t)2 * C * c.post_merge_dim, (size_t)2 * C,
                           (size_t)C * 3 * C};
      size_t total = 0;
      for (size_t k : n) total += (k + 63) & ~(size_t)63;      // 256-byte aligned pieces
      LVSR_CUDA_OK(s.mem.alloc(total * sizeof(float)));
      float** piece[4] = {&s.Ws, &s.Wm, &s.h0, &s.F};
      float* p = s.mem.get();
      for (int i = 0; i < 4; ++i) { *piece[i] = p; p += (n[i] + 63) & ~(size_t)63; }
    }
    m->Wcat = std::move(Wcat);
    m->bcat = std::move(bcat);
    for (int l = 0; l < 2; ++l) m->dec[l] = std::move(dec[l]);
    m->Wb1 = std::move(Wb1);
    m->stack = std::move(s);
  }
  for (int l = 0; l < c.num_layers; ++l)
    for (int dir = 0; dir < encoder_dirs(m); ++dir)
      if (int rc = fork_copy(m, encoder_fork(m, l, dir), m->Wcat[l].get(), m->bcat[l].get(), nullptr, st)) return rc;
  const int C = c.dim_dec, Cfb = c.dim_feedback, V = c.num_phonemes;
  const std::string g = GEN, t = TR;
  // decoder-side packing, per layer: gate columns first (update | reset), then the candidate inputs
  for (int l = 0; l < c.dec_stack; ++l) {
    const lvsr_model::DecLayer& d = m->dec[l];
    const std::string x = layer_suffix(l);
    const std::string dist = t + "/distribute/";
    float *Wd = d.Wd.get(), *Wff = d.Wff.get(), *bff = d.bff.get(), *FF = d.FF.get();
    if (int rc = copy2d(Wd, 3 * C, m->P(dist + "fork_gate_inputs" + x + ".W"), 2 * C, m->E, 2 * C, st)) return rc;
    if (int rc = copy2d(Wd + 2 * C, 3 * C, m->P(dist + "fork_inputs" + x + ".W"), C, m->E, C, st)) return rc;
    if (int rc = fork_copy(m, feedback_fork(c, l), Wff, bff, nullptr, st)) return rc;
    // fork(feedback(y)) for every symbol y, once: [(V+1), 3C]
    if (c.one_of_n_feedback) {
      // one-hot feedback: fork(feedback(y)) is row y of the fork weights plus the bias
      if (int rc = add_bias_rows(FF, Wff, bff, V + 1, 3 * C, st)) return rc;
    } else {
      GemmArgs ff = make_gemm(m->P(g + "/readout/lookupfeedback/lookuptable.W"), V + 1, Cfb, Wff, 3 * C, bff, FF);
      if (int rc = gemm_bias(ff, st)) return rc;
    }
  }
  LVSR_CUDA_OK(cudaMemsetAsync(m->Wb1.get(), 0, (size_t)(m->E + C) * 3 * C * sizeof(float), st));
  if (int rc = copy2d(m->Wb1.get(), 3 * C, m->dec[0].Wd.get(), 3 * C, m->E, 3 * C, st)) return rc;
  if (int rc = copy2d(m->Wb1.get() + (size_t)m->E * 3 * C, 3 * C, m->P(dec_gru(m, 0) + ".state_to_gates"), 2 * C, C, 2 * C, st)) return rc;
  // tensor-core operands of the fork and preprocess weights (K-major fp16 head/tail planes or tf32 hi/lo pairs)
  m->use_tc = getenv("LVSR_NO_TC_GEMM") == nullptr;
  if (m->use_tc) {
    m->Wcat_tc.resize(c.num_layers);
    for (int l = 0; l < c.num_layers; ++l) {
      const ForkLayout f = encoder_fork(m, l, 0);
      if (int rc = pack_tc_weights(m->Wcat_tc[l], m->Wcat[l].get(), f.rows, f.ld, st)) return rc;
    }
    if (int rc = pack_tc_weights(m->Wp_tc, m->P(att_base(m) + "/preprocess.W"), m->E, c.dim_matcher, st)) return rc;
    m->bottom_tc.resize(m->bottom.num_layers);
    for (int i = 0; i < m->bottom.num_layers; ++i)
      if (int rc = pack_tc_weights(m->bottom_tc[i], m->P(bottom_linear(i) + ".W"), bottom_input_dim(m, i), m->bottom.dims[i],
                                   st))
        return rc;
  }
  if (c.dec_stack == 2) {
    // the wide state's row-stacked weights [W ; W#1], both initial states, and fork_1 of layer 0's new state
    lvsr_model::Stack& s = m->stack;
    const int M = c.dim_matcher, Cpm = c.post_merge_dim;
    const std::string a = att_base(m), r = t + "/recurrentstack";
    if (int rc = copy2d(s.Ws, M, m->P(a + "/state_trans/transform_states.W"), M, C, M, st)) return rc;
    if (int rc = copy2d(s.Ws + (size_t)C * M, M, m->P(a + "/state_trans/transform_states#1.W"), M, C, M, st)) return rc;
    if (c.use_states_for_readout) {
      if (int rc = copy2d(s.Wm, Cpm, m->P(g + "/readout/merge/transform_states.W"), Cpm, C, Cpm, st)) return rc;
      if (int rc = copy2d(s.Wm + (size_t)C * Cpm, Cpm, m->P(g + "/readout/merge/transform_states#1.W"), Cpm, C, Cpm, st))
        return rc;
    }
    if (int rc = copy2d(s.h0, C, m->P(dec_gru(m, 0) + ".initial_state"), C, 1, C, st)) return rc;
    if (int rc = copy2d(s.h0 + C, C, m->P(dec_gru(m, 1) + ".initial_state"), C, 1, C, st)) return rc;
    if (int rc = copy2d(s.F, 3 * C, m->P(r + "/fork_1/fork_gate_inputs.W"), 2 * C, C, 2 * C, st)) return rc;
    if (int rc = copy2d(s.F + 2 * C, 3 * C, m->P(r + "/fork_1/fork_inputs.W"), C, C, C, st)) return rc;
  }
  m->v_bias = 0.f;
  if (c.energy_normalizer != LVSR_NORM_SOFTMAX) {
    // a kernel argument: read in st's order (after an update enqueued there), so the host waits for st
    LVSR_CUDA_OK(cudaMemcpyAsync(&m->v_bias, m->P(att_base(m) + "/energy_comp/linear.b"), sizeof(float),
                                 cudaMemcpyDeviceToHost, st));
    LVSR_CUDA_OK(cudaStreamSynchronize(st));
  }
  if (synchronise) LVSR_CUDA_OK(cudaStreamSynchronize(st));
  m->finalized = true;
  return 0;
}

// out[M, N] = A[M, K] . W + bias: the wgmma GEMM when W has a tensor-core form (tw, packed by finalize) and the shape
// suits it, else the FFMA tile GEMM.  The operand kind follows K: fp16 head/tail (f16x3) when K is a multiple of 64, so
// every encoder layer from 1 on and the preprocess, 3xTF32 with K padded to a multiple of 32 otherwise (layer 0 at 40
// features).  The split of A is scratch taken from `ws` and left there: it is dead once the GEMM is enqueued, and the
// caller decides when to rewind it (lvsr_cost_matrix allocates the persistent decoder's buffers behind it, and their
// place in the workspace is part of the decoder's measured step time).  Both kinds take the same 2 M kpad(K) floats,
// so that place does not depend on the kind: the fp16 planes (M K halves each) fill the first half, the row exponents
// sit at the start of the second.
int projection_gemm(Arena& ws, const float* A, int M, int K, const float* W, const TcWeights* tw, int N,
                    const float* bias, float* out, cudaStream_t st, int* kpad, int* operands) {
  const bool f16 = tw && tw->head && gemm_f16_supported(M, N, K);
  const bool tf32 = tw && tw->hi && gemm_tc_supported(M, N, K);
  if (f16 || tf32) {
    float* a_hi = ws.f32((size_t)M * gemm_tc_kpad(K));
    float* a_lo = ws.f32((size_t)M * gemm_tc_kpad(K));
    LVSR_CHECK(a_hi && a_lo, "out of device memory (tensor-core split scratch)");
    if (kpad) *kpad = gemm_tc_kpad(K);
    if (operands) *operands = f16 ? LVSR_ENC_OPS_F16X3 : LVSR_ENC_OPS_TF32X3;
    if (f16) {
      __half* a_head = reinterpret_cast<__half*>(a_hi);
      return gemm_f16(A, a_head, a_head + (size_t)M * K, reinterpret_cast<int*>(a_lo), M, K, tw->head, tw->tail, tw->ew,
                      N, bias, out, N, st);
    }
    return gemm_tc(A, a_hi, a_lo, M, K, tw->hi, tw->lo, N, bias, out, N, st);
  }
  if (kpad) *kpad = 0;
  if (operands) *operands = LVSR_ENC_OPS_NONE;
  return gemm_bias(make_gemm(A, M, K, W, N, bias, out), st);
}

// The SMs a scan must leave free for the projection behind it to run beside it (api.cu: run_encoder)
constexpr int ENC_OVERLAP_MIN_SMS = 16;

int run_encoder(lvsr_model* m, Arena& ws, const float* x, const float* mask, int T, int B, float* attended,
                float* attended_mask, LayerTape* tape, cudaStream_t st, const float** bottom_out,
                const DropoutKey* dropout) {
  const lvsr_config& c = m->cfg;
  const float* cur = x;
  int Tl = T, din = encoder_input_dim(m);
  if (m->bottom.num_layers) {
    // every frame, padded ones included: the BiGRU's mask keeps them out of the states and their gradients
    const float* y[LVSR_MAX_BOTTOM] = {};
    if (int rc = bottom_forward(m, ws, x, T * B, y, st)) return rc;
    cur = y[m->bottom.num_layers - 1];
    if (bottom_out)
      for (int i = 0; i < m->bottom.num_layers; ++i) bottom_out[i] = y[i];
  }
  if (dropout) {
    float* dropped = ws.f32((size_t)T * B * din);
    LVSR_CHECK(dropped, "out of device memory (dropout)");
    if (int rc = dropout_apply(*dropout, cur, dropped, T, B, din, st)) return rc;
    cur = dropped;
  }
  long long mstride = B;
  int kcum = 1;
  for (int l = 0; l < c.num_layers; ++l) {
    for (int s = LVSR_ENC_PROJ; s <= LVSR_ENC_T; ++s) m->enc_plan[l][s] = 0;
    m->enc_plan[l][LVSR_ENC_OPERANDS] = 0;
    m->enc_overlap[l] = 0;
  }
  // LVSR_ENC_OVERLAP=0: every projection after the scan before it; LVSR_ENC_OVERLAP_SPIN_LIMIT: polls without scan
  // progress after which the projection beside a scan stops claiming tiles (0: at its first tile that is not final)
  const char* ov = getenv("LVSR_ENC_OVERLAP");
  const bool overlap_on = m->use_tc && !(ov && atoi(ov) == 0);
  const char* sl = getenv("LVSR_ENC_OVERLAP_SPIN_LIMIT");
  const unsigned spin_limit = sl ? (unsigned)strtoul(sl, nullptr, 10) : LVSR_SPIN_LIMIT;
  if (overlap_on && c.num_layers > 1) {
    if (!m->enc_tiles) LVSR_CUDA_OK(m->enc_tiles.alloc(LVSR_MAX_LAYERS * 2 * sizeof(int)));
    LVSR_CUDA_OK(cudaMemsetAsync(m->enc_tiles.get(), 0, LVSR_MAX_LAYERS * 2 * sizeof(int), st));
    // the claim records of every layer's projection (lvsr_model_encoder_overlap_claims)
    size_t need = 0;
    for (int l = 1, Tp = ceil_div(T, c.subsample[0]); l < c.num_layers; Tp = ceil_div(Tp, c.subsample[l]), ++l) {
      m->enc_claims_off[l] = need;
      need += 3 * (size_t)ceil_div(Tp * B, 128) * (encoder_fork(m, l, 0).ld / 128);
    }
    LVSR_CUDA_OK(m->enc_claims.grow(need * sizeof(int), st));
    LVSR_CUDA_OK(cudaMemsetAsync(m->enc_claims.get(), 0, need * sizeof(int), st));
  }
  float* pre_done = nullptr;   // this layer's pre-activations, when they were projected beside the previous scan
  const int nd = encoder_dirs(m);
  for (int l = 0; l < c.num_layers; ++l) {
    const int D = c.dims_bidir[l], k = c.subsample[l], N = encoder_fork(m, l, 0).ld, Dout = encoder_output_dim(m, l);
    const int rows = Tl * B, Tout = ceil_div(Tl, k);
    float* pre = pre_done ? pre_done : ws.f32((size_t)rows * N);
    float* hext = tape ? ws.f32((size_t)(Tl + 2) * B * Dout) : nullptr;
    LVSR_CHECK(pre && (hext || !tape), "out of device memory (encoder pre-activations)");
    int32_t* plan = m->enc_plan[l];
    if (!pre_done) {
      // finalize splits the fork weights only while the tensor-core GEMM is on (null entry: a shape it refuses)
      ArenaMark mark{ws};      // the split scratch is dead once the GEMM is enqueued (stream order)
      int kpad = 0, operands = 0;
      if (int rc = projection_gemm(ws, cur, rows, din, m->Wcat[l].get(), m->use_tc ? &m->Wcat_tc[l] : nullptr, N, m->bcat[l].get(),
                                   pre, st, &kpad, &operands))
        return rc;
      plan[LVSR_ENC_PROJ] = kpad ? LVSR_ENC_PATH_TC : LVSR_ENC_PATH_FFMA;
      plan[LVSR_ENC_KPAD] = kpad;
      plan[LVSR_ENC_OPERANDS] = operands;
    }
    pre_done = nullptr;
    float* out = (l == c.num_layers - 1) ? attended : ws.f32((size_t)Tout * B * Dout);
    LVSR_CHECK(out, "out of device memory (encoder layer output)");
    BiGruArgs a = {};
    a.pre = pre; a.mask = mask; a.mask_tstride = mstride;
    const std::string bf = enc_base(m, l, 0) + "/gatedrecurrent", bb = enc_base(m, l, 1) + "/gatedrecurrent";
    a.Wg_f = m->P(bf + ".state_to_gates"); a.Ws_f = m->P(bf + ".state_to_state"); a.h0_f = m->P(bf + ".initial_state");
    if (nd == 2) {
      a.Wg_b = m->P(bb + ".state_to_gates"); a.Ws_b = m->P(bb + ".state_to_state"); a.h0_b = m->P(bb + ".initial_state");
    }
    a.out = out; a.T = Tl; a.B = B; a.D = D; a.subsample = k; a.ndir = nd;
    if (tape) {
      a.tape = pre; a.hext = hext;
      tape[l] = {cur, pre, hext, Tl, din, D, k, mstride};
    }
    // Layer l + 1's projection reads only this scan's output: its tiles can run beside the scan, on the SMs the scan
    // leaves idle, as their rows become final -- when the scan runs in one wave of tensor-core clusters that leaves
    // ENC_OVERLAP_MIN_SMS free and the projection takes fp16 operands
    BiGruPlan bp;
    if (int rc = bigru_plan(a, &bp)) return rc;
    const int scan_ctas = bp.clusters * bp.cs, free_sms = device_sm_count() - scan_ctas;
    const int l1 = l + 1, N1 = l1 < c.num_layers ? encoder_fork(m, l1, 0).ld : 0, rows1 = Tout * B;
    const bool overlap = overlap_on && l1 < c.num_layers && bp.kernel == LVSR_ENC_BIGRU_MMA && bp.waves == 1 &&
                         free_sms >= ENC_OVERLAP_MIN_SMS && scan_ctas <= gemm_f16_stream_max_scan_ctas() &&
                         m->Wcat_tc[l1].head && gemm_f16_stream_supported(rows1, N1, Dout);
    if (!overlap) {
      ProfScope prof("bigru", st);
      if (int rc = bigru_layer(a, st, &bp)) return rc;
    } else {
      // the same arena order as without the overlap (pre-activations of l + 1 right after this layer's output), the
      // split planes as projection_gemm takes them, then the scheduling area; all but the pre-activations dead after
      float* pre1 = ws.f32((size_t)rows1 * N1);
      ArenaMark mark{ws};
      const int K1 = Dout;
      float* a_hi = ws.f32((size_t)rows1 * K1);
      float* a_lo = ws.f32((size_t)rows1 * K1);
      int* sync = reinterpret_cast<int*>(ws.f32(gemm_f16_stream_sync_ints(rows1)));
      LVSR_CHECK(pre1 && a_hi && a_lo && sync, "out of device memory (streamed projection)");
      LVSR_CUDA_OK(cudaMemsetAsync(sync, 0, gemm_f16_stream_sync_ints(rows1) * sizeof(int), st));
      a.progress = gemm_f16_stream_progress(sync);
      __half* a_head = reinterpret_cast<__half*>(a_hi);
      const TcWeights& tw = m->Wcat_tc[l1];
      ProjStream ps = {sync, a.progress, scan_ctas, bp.cs, nd, Tl, k, B, spin_limit, m->enc_tiles.get() + 2 * l1,
                       m->enc_claims.get() + m->enc_claims_off[l1]};
      {
        // no event between the two launches: the projection must directly follow the scan in the stream.  The
        // profiled "bigru" time therefore covers the scan and the projection tiles done beside it.
        ProfScope prof("bigru", st);
        if (int rc = bigru_layer(a, st, &bp)) return rc;
        if (int rc = gemm_f16_stream(out, a_head, a_head + (size_t)rows1 * K1, reinterpret_cast<int*>(a_lo), rows1, K1,
                                     tw.head, tw.tail, tw.ew, N1, m->bcat[l1].get(), pre1, N1, ps, free_sms, st))
          return rc;
      }
      {
        ProfScope prof("gemm", st);
        ps.progress = nullptr;
        ps.tiles_done = m->enc_tiles.get() + 2 * l1 + 1;
        if (int rc = gemm_f16_stream(out, a_head, a_head + (size_t)rows1 * K1, reinterpret_cast<int*>(a_lo), rows1, K1,
                                     tw.head, tw.tail, tw.ew, N1, m->bcat[l1].get(), pre1, N1, ps, device_sm_count(), st))
          return rc;
      }
      int32_t* plan1 = m->enc_plan[l1];
      plan1[LVSR_ENC_PROJ] = LVSR_ENC_PATH_TC;
      plan1[LVSR_ENC_KPAD] = K1;
      plan1[LVSR_ENC_OPERANDS] = LVSR_ENC_OPS_F16X3;
      m->enc_overlap[l1] = 1;
      pre_done = pre1;
    }
    plan[LVSR_ENC_BIGRU] = bp.kernel;
    plan[LVSR_ENC_TAPE] = tape ? 1 : 0;
    plan[LVSR_ENC_RB] = bp.rb;
    plan[LVSR_ENC_CS] = bp.cs;
    plan[LVSR_ENC_CLUSTERS] = bp.clusters;
    plan[LVSR_ENC_RESIDENT] = bp.resident;
    plan[LVSR_ENC_WAVES] = bp.waves;
    plan[LVSR_ENC_T] = Tl;
    cur = out; Tl = Tout; din = Dout; mstride *= k; kcum *= k;
  }
  if (mask) {
    if (int rc = gather_time_subsample(attended_mask, mask, Tl, kcum, B, st)) return rc;
  } else {
    if (int rc = fill_f32(attended_mask, (long long)Tl * B, 1.f, st)) return rc;   // lvsr/bricks/__init__.py:78
  }
  return 0;
}
}  // namespace lvsr

// Workspace of tle_costs
static size_t tle_ws_bytes(const lvsr_model* m, int Lg, int L, int B) {
  return (size_t)3 * L * B * m->cfg.num_phonemes * sizeof(float) + tle_dist_ints(Lg, L, B) * sizeof(int) + 4096;
}

int lvsr::tle_check_status(lvsr_model* m, cudaStream_t st) {
  unsigned h = LVSR_TLE_OK;
  LVSR_CUDA_OK(cudaMemcpyAsync(&h, m->tle_status.get(), sizeof(h), cudaMemcpyDeviceToHost, st));
  LVSR_CUDA_OK(cudaStreamSynchronize(st));
  LVSR_CHECK(h == LVSR_TLE_OK, "task loss estimation: the groundtruth of utterance %u does not end in eos (%d)", h,
             m->criterion.eos_label);
  return 0;
}

// RewardOp's matrices of prediction [L, B] against groundtruth [Lg, B] into rewards / gains [L, B, V] (from ws); with
// `wait`, synchronises st and reports the first utterance whose groundtruth holds no eos (else tle_check_status does)
static int tle_run_matrices(lvsr_model* m, Arena& ws, const long long* groundtruth, int Lg, const long long* prediction,
                            int L, int B, float* rewards, float* gains, bool wait, cudaStream_t st) {
  int* dist = ws.i32(tle_dist_ints(Lg, L, B));
  LVSR_CHECK(dist, "out of device memory (task-loss distances)");
  LVSR_CUDA_OK(cudaMemsetAsync(m->tle_status.get(), 0xff, sizeof(unsigned), st));
  if (int rc = tle_matrices(groundtruth, Lg, prediction, L, B, m->cfg.num_phonemes, m->criterion.eos_label, dist, rewards,
                            gains, m->tle_status.get(), st)) return rc;
  return wait ? tle_check_status(m, st) : 0;
}

// The task-loss cost rows [L, B] from the emitter costs neg [L*B, V] of the prediction `labels`; the matrices go to
// keep's buffers when it is given
static int tle_costs(lvsr_model* m, Arena& ws, const long long* groundtruth, int Lg, const long long* labels,
                     const float* lmask, int L, int B, const float* neg, float* costs, const TleTape* keep,
                     cudaStream_t st) {
  const size_t n = (size_t)L * B * m->cfg.num_phonemes;
  float* rewards = keep ? keep->rewards : ws.f32(n);
  float* gains = keep ? keep->gains : ws.f32(n);
  LVSR_CHECK(rewards && gains, "out of device memory (task-loss matrices)");
  if (int rc = tle_run_matrices(m, ws, groundtruth, Lg, labels, L, B, rewards, gains, !keep, st)) return rc;
  const int loss = m->criterion.name == LVSR_CRITERION_MSE_GAIN ? LVSR_TLE_GAIN : LVSR_TLE_REWARD;
  return tle_loss(loss, neg, rewards, gains, labels, lmask, L, B, m->cfg.num_phonemes, (float)m->criterion.min_reward,
                  costs, st);
}

extern "C" {

int lvsr_model_set_criterion(lvsr_model* m, const lvsr_criterion* cr) {
  DeviceGuard device_guard(m);
  LVSR_CHECK(m && cr, "set_criterion: bad arguments");
  const int V = m->cfg.num_phonemes;
  LVSR_CHECK(cr->name == LVSR_CRITERION_LOG_LIKELIHOOD || cr->name == LVSR_CRITERION_MSE_GAIN ||
                 cr->name == LVSR_CRITERION_MSE_REWARD, "set_criterion: unknown criterion %d", cr->name);
  if (cr->name != LVSR_CRITERION_LOG_LIKELIHOOD) {
    LVSR_CHECK(cr->eos_label >= 0 && cr->eos_label < V, "set_criterion: eos_label %d outside [0, %d)", cr->eos_label, V);
    LVSR_CHECK(cr->initial_output >= 0 && cr->initial_output <= V, "set_criterion: initial_output %d outside [0, %d]",
               cr->initial_output, V);
    LVSR_CHECK(std::isfinite(cr->min_reward), "set_criterion: min_reward must be finite");
    if (!m->tle_status) LVSR_CUDA_OK(m->tle_status.alloc(sizeof(unsigned)));
  }
  LVSR_CUDA_OK(cudaStreamSynchronize(m->stream));   // calls already queued keep the criterion they were issued under
  m->criterion = *cr;
  return 0;
}

int lvsr_tle_matrices(lvsr_model* m, const int64_t* groundtruth, int32_t Lg, const int64_t* prediction, int32_t L,
                      int32_t B, float* rewards, float* gains, void* stream) {
  DeviceGuard device_guard(m);
  if (int rc = bind_stream(m, static_cast<cudaStream_t>(stream))) return rc;
  LVSR_CHECK(groundtruth && prediction && rewards && gains && Lg > 0 && L > 0 && B > 0, "tle_matrices: bad arguments");
  LVSR_CHECK(tle_criterion(m), "tle_matrices: the handle's criterion is log_likelihood (lvsr_model_set_criterion)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  m->ws.reserve(tle_ws_bytes(m, Lg, L, B), st);
  ArenaScope scope(m, st);
  return tle_run_matrices(m, m->ws, reinterpret_cast<const long long*>(groundtruth), Lg,
                          reinterpret_cast<const long long*>(prediction), L, B, rewards, gains, true, st);
}

int lvsr_encoded_length(const lvsr_model* m, int32_t T) {
  if (!m) return 0;
  int t = T;
  for (int l = 0; l < m->cfg.num_layers; ++l) t = ceil_div(t, m->cfg.subsample[l]);
  return t;
}
int lvsr_encoded_dim(const lvsr_model* m) { return m ? m->E : 0; }

int lvsr_encoder_forward(lvsr_model* m, const float* x, const float* mask, int32_t T, int32_t B,
                         float* attended, float* attended_mask, void* stream) {
  DeviceGuard device_guard(m);
  if (int rc = bind_stream(m, static_cast<cudaStream_t>(stream))) return rc;
  if (int rc = check_ready(m)) return rc;
  LVSR_CHECK(x && attended && attended_mask && T > 0 && B > 0, "encoder_forward: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  m->ws.reserve(encoder_ws_bytes(m, T, B), st);
  ArenaScope scope(m, st);
  return run_encoder(m, m->ws, x, mask, T, B, attended, attended_mask, nullptr, st);
}

int lvsr_preprocess(lvsr_model* m, const float* attended, int32_t Tp, int32_t U, float* out, void* stream) {
  DeviceGuard device_guard(m);
  if (int rc = bind_stream(m, static_cast<cudaStream_t>(stream))) return rc;
  if (int rc = check_ready(m)) return rc;
  LVSR_CHECK(attended && out && Tp > 0 && U > 0, "preprocess: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ArenaScope scope(m, st);
  int kpad = 0, operands = 0;
  m->pre_plan[0] = m->pre_plan[1] = m->pre_plan[2] = 0;
  if (int rc = projection_gemm(m->ws, attended, Tp * U, m->E, m->P(att_base(m) + "/preprocess.W"),
                               m->use_tc ? &m->Wp_tc : nullptr, m->cfg.dim_matcher, m->P(att_base(m) + "/preprocess.b"),
                               out, st, &kpad, &operands))
    return rc;
  m->pre_plan[0] = kpad ? LVSR_ENC_PATH_TC : LVSR_ENC_PATH_FFMA;
  m->pre_plan[1] = kpad;
  m->pre_plan[2] = operands;
  return 0;
}

int lvsr_cost_matrix(lvsr_model* m, const float* attended, const float* attended_mask, int32_t Tp, int32_t B,
                     const int64_t* labels, const float* labels_mask, int32_t L, float* costs,
                     float* weights_out, float* energies_out, float* states_out, float* wavg_out, void* stream) {
  return lvsr_cost_matrix_groundtruth(m, attended, attended_mask, Tp, B, labels, labels_mask, L, nullptr, 0, costs,
                                      weights_out, energies_out, states_out, wavg_out, stream);
}

int lvsr_cost_matrix_groundtruth(lvsr_model* m, const float* attended, const float* attended_mask, int32_t Tp, int32_t B,
                                 const int64_t* labels, const float* labels_mask, int32_t L, const int64_t* groundtruth,
                                 int32_t Lg, float* costs, float* weights_out, float* energies_out, float* states_out,
                                 float* wavg_out, void* stream) {
  return cost_matrix(m, attended, attended_mask, Tp, B, labels, labels_mask, L, groundtruth, Lg, costs, weights_out,
                     energies_out, states_out, wavg_out, nullptr, static_cast<cudaStream_t>(stream));
}

}  // extern "C"

int lvsr::cost_matrix(lvsr_model* m, const float* attended, const float* attended_mask, int Tp, int B,
                      const int64_t* labels, const float* labels_mask, int L, const int64_t* groundtruth, int Lg,
                      float* costs, float* weights_out, float* energies_out, float* states_out, float* wavg_out,
                      const TleTape* keep, cudaStream_t st) {
  DeviceGuard device_guard(m);
  if (int rc = bind_stream(m, st)) return rc;
  if (int rc = check_ready(m)) return rc;
  LVSR_CHECK(attended && attended_mask && labels && costs && Tp > 0 && B > 0 && L > 0, "cost_matrix: bad arguments");
  LVSR_CHECK(!groundtruth || Lg > 0, "cost_matrix: groundtruth without rows");
  const bool tle = tle_criterion(m);
  if (!groundtruth) { groundtruth = labels; Lg = L; }
  m->ws.reserve(cost_ws_bytes(m, Tp, B, L) + (lm_attached(m) ? (size_t)L * B * m->cfg.num_phonemes * sizeof(float) : 0) +
                    (tle ? tle_ws_bytes(m, Lg, L, B) : 0), st);
  ArenaScope scope(m, st);
  const lvsr_config& c = m->cfg;
  Arena& ws = m->ws;
  const int C = c.dim_dec, E = m->E, M = c.dim_matcher, S = state_dim(m);
  const long long* lab = reinterpret_cast<const long long*>(labels);

  float* P = ws.f32((size_t)Tp * B * M);
  float* s_all = ws.f32((size_t)(L + 1) * B * S);
  float* ctx_all = wavg_out ? wavg_out : ws.f32((size_t)L * B * E);
  float* w0 = ws.f32((size_t)B * Tp);
  float* wpp[2] = {ws.f32((size_t)B * Tp), ws.f32((size_t)B * Tp)};   // step-wise fallback only
  float* e_scratch = energies_out ? nullptr : ws.f32((size_t)B * Tp);
  float* merged = ws.f32((size_t)L * B * c.post_merge_dim);
  LVSR_CHECK(P && s_all && ctx_all && w0 && merged && wpp[0] && wpp[1] && (energies_out || e_scratch),
             "out of device memory (decoder workspace)");

  if (int rc = lvsr_preprocess(m, attended, Tp, B, P, st)) return rc;              // hoisted: B/bricks/attention.py:733-738
  if (int rc = broadcast_rows(s_all, initial_state_row(m), B, S, st)) return rc;
  if (int rc = onehot_rows(w0, B, Tp, st)) return rc;                               // lvsr/bricks/attention.py:215-222
  if (int rc = fill_f32(costs, (long long)L * B, 0.f, st)) return rc;

  bool scanned = false;
  for (int32_t& v : m->dec_plan) v = 0;
  LVSR_CUDA_OK(cudaMemsetAsync(m->status.get(), 0, sizeof(unsigned), st));
  // the persistent decoder holds one GRU layer: a stacked decoder runs on the step-wise kernels
  if (getenv("LVSR_NO_DEC_SCAN") == nullptr && !m->force_stepwise && c.dec_stack == 1) {
    DecScanInputs d = {};
    d.P = P; d.H = attended; d.maskH = attended_mask;
    d.filt = m->P(att_base(m) + "/conv1d.filters");     // null for content attention
    d.Wh = m->P(att_base(m) + "/handler.W");
    d.v = m->P(att_base(m) + "/energy_comp/linear.W");
    d.v_bias = m->v_bias;
    d.prior = prior_of(c);
    d.Wb1 = m->Wb1.get();
    d.Wstate = m->P(dec_gru(m, 0) + ".state_to_state");
    d.Ws = m->P(att_base(m) + "/state_trans/transform_states.W");
    d.FF = m->dec[0].FF.get();
    d.labels = lab; d.lmask = labels_mask;
    d.s_all = s_all; d.ctx_all = ctx_all; d.w0 = w0; d.w_all = weights_out;
    d.e_seq = energies_out; d.e_scratch = e_scratch;
    d.status = m->status.get();
    d.Tp = Tp; d.B = B; d.L = L; d.M = M; d.E = E; d.C = C; d.K = c.conv_num_filters; d.n = c.conv_n;
    d.normalizer = c.energy_normalizer;
    d.V = c.num_phonemes;
    // the persistent decoder's buffers follow `merged` and the preprocess's split scratch in the workspace
    if (int rc = run_dec_scan(d, !content_attention(m), ws, m->dec_plan, &scanned, st)) return rc;
  }
  const float* w_prev = w0;
  for (int i = 0; i < L && !scanned; ++i) {
    float* w_i = weights_out ? weights_out + (size_t)i * B * Tp : wpp[i & 1];
    float* e_i = energies_out ? energies_out + (size_t)i * B * Tp : e_scratch;
    float* ctx_i = ctx_all + (size_t)i * B * E;
    const float* s_i = s_all + (size_t)i * B * S;
    ArenaMark mark{ws};   // per-step scratch is reusable (stream order): rewound at the end of every step
    if (int rc = glimpses(m, attended, P, attended_mask, Tp, B, nullptr, B, s_i, w_prev, nullptr, i, w_i, e_i, ctx_i, st)) return rc;
    if (int rc = transition(m, B, s_i, ctx_i, lab + (size_t)i * B, labels_mask ? labels_mask + (size_t)i * B : nullptr,
                            s_all + (size_t)(i + 1) * B * S, st)) return rc;
    w_prev = w_i;
  }
  // the language model's cost rows in force before each label (sequence_generators.py:284-289), then fused below
  float* lm_add = nullptr;
  if (lm_attached(m)) {
    lm_add = ws.f32((size_t)L * B * c.num_phonemes);
    LVSR_CHECK(lm_add, "out of device memory (language model costs)");
    if (int rc = lm_path(lm_fst(m), L, B, lab, labels_mask, lm_add, st)) return rc;
    if (int rc = lm_sync_status(m, st)) return rc;
  }
  // readout(states[:-1], glimpses[1:]) for all steps at once, then the emitter cost
  {
    const int R = L * B;
    const std::string g = GEN;
    bool acc = false;
    if (c.use_states_for_readout) {
      GemmArgs a = make_gemm(s_all, R, S, readout_state_weights(m), c.post_merge_dim, nullptr, merged);
      if (int rc = gemm_bias(a, st)) return rc;
      acc = true;
    }
    GemmArgs b = make_gemm(ctx_all, R, E, m->P(g + "/readout/merge/transform_weighted_averages.W"), c.post_merge_dim,
                           nullptr, merged, acc);
    if (readout_depth(m) > 1) {          // h_0 = act(merge + post_merge/bias.b) in the merge's epilogue
      b.bias = m->P(g + "/readout/post_merge/bias.b");
      b.act = c.post_merge_activation;
    }
    if (int rc = gemm_bias(b, st)) return rc;
    const float* tail = nullptr;
    if (int rc = readout_body(m, ws, R, merged, true, &tail, nullptr, st)) return rc;
    ReadoutArgs r = readout_args(m, R, tail);
    r.poison = scanned ? m->status.get() : nullptr;
    if (lm_add) lm_fuse(m, r, lm_add);
    if (tle) {
      // RewardRegressionEmitter.cost over the whole readouts (lvsr/bricks/__init__.py:135-184); with a language model
      // these are the fused readouts x, whose LM rows follow the labels (the prediction), not the groundtruth
      float* neg = keep ? keep->neg : ws.f32((size_t)R * c.num_phonemes);
      LVSR_CHECK(neg, "out of device memory (task-loss readouts)");
      r.costs_all = neg;
      if (int rc = readout_costs(r, st)) return rc;
      if (int rc = tle_costs(m, ws, reinterpret_cast<const long long*>(groundtruth), Lg, lab, labels_mask, L, B, neg,
                             costs, keep, st)) return rc;
    } else {
      r.labels = lab; r.lmask = labels_mask; r.costs_picked = costs;
      if (int rc = readout_costs(r, st)) return rc;
    }
  }
  if (states_out)
    LVSR_CUDA_OK(cudaMemcpyAsync(states_out, s_all, (size_t)L * B * S * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

int lvsr::tle_generate_greedy(lvsr_model* m, const float* attended, const float* attended_mask, int Tp, int B, int n,
                              long long* prediction, float* prediction_mask, cudaStream_t st) {
  ProfScope prof("tle_generate", st);
  const lvsr_config& c = m->cfg;
  const int E = m->E, S = state_dim(m), V = c.num_phonemes;
  m->ws.reserve(cost_ws_bytes(m, Tp, B, 1), st);
  ArenaScope scope(m, st);
  Arena& ws = m->ws;
  float* P = ws.f32((size_t)Tp * B * c.dim_matcher);
  float* s[2] = {ws.f32((size_t)B * S), ws.f32((size_t)B * S)};
  float* w[2] = {ws.f32((size_t)B * Tp), ws.f32((size_t)B * Tp)};
  float* e = ws.f32((size_t)B * Tp);
  float* ctx = ws.f32((size_t)B * E);
  float* merged = ws.f32((size_t)B * c.post_merge_dim);
  float* neg = ws.f32((size_t)B * V);
  float* alive = ws.f32((size_t)B);
  LVSR_CHECK(P && s[0] && s[1] && w[0] && w[1] && e && ctx && merged && neg && alive,
             "out of device memory (greedy generation)");
  if (int rc = lvsr_preprocess(m, attended, Tp, B, P, st)) return rc;
  if (int rc = broadcast_rows(s[0], initial_state_row(m), B, S, st)) return rc;
  if (int rc = onehot_rows(w[0], B, Tp, st)) return rc;
  if (int rc = fill_f32(alive, B, 1.f, st)) return rc;
  for (int i = 0; i < n; ++i) {
    ArenaMark mark{ws};
    const float* s_i = s[i & 1];
    if (int rc = glimpses(m, attended, P, attended_mask, Tp, B, nullptr, B, s_i, w[i & 1], nullptr, i, w[(i + 1) & 1], e,
                          ctx, st)) return rc;
    const float* tail = nullptr;
    if (int rc = readout_merged(m, B, s_i, ctx, merged, &tail, st)) return rc;
    ReadoutArgs r = readout_args(m, B, tail);
    r.costs_all = neg;
    if (int rc = readout_costs(r, st)) return rc;
    long long* y_i = prediction + (size_t)i * B;
    if (int rc = tle_greedy_pick(neg, B, V, m->criterion.eos_label, alive, y_i, prediction_mask + (size_t)i * B, st)) return rc;
    if (int rc = transition(m, B, s_i, ctx, y_i, nullptr, s[(i + 1) & 1], st)) return rc;
  }
  return 0;
}

extern "C" {

int lvsr_initial_states(lvsr_model* m, int32_t Tp, int32_t R, float* states, int64_t* outputs, float* wavg,
                        float* weights, float* energies, int64_t* step, void* stream) {
  DeviceGuard device_guard(m);
  if (int rc = bind_stream(m, static_cast<cudaStream_t>(stream))) return rc;
  if (int rc = check_ready(m)) return rc;
  LVSR_CHECK(states && outputs && wavg && weights && energies && step && Tp > 0 && R > 0, "initial_states: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = broadcast_rows(states, initial_state_row(m), R, state_dim(m), st)) return rc;
  if (int rc = fill_i64(reinterpret_cast<long long*>(outputs), R, initial_output(m), st)) return rc;
  if (int rc = fill_f32(wavg, (long long)R * m->E, 0.f, st)) return rc;
  if (content_attention(m)) {             // B/bricks/attention.py:392-395: zero weights; no energies state
    if (int rc = fill_f32(weights, (long long)R * Tp, 0.f, st)) return rc;
    if (int rc = fill_f32(energies, (long long)R * Tp, 0.f, st)) return rc;
  } else {
    if (int rc = onehot_rows(weights, R, Tp, st)) return rc;
    if (int rc = onehot_rows(energies, R, Tp, st)) return rc;
  }
  return fill_i64(reinterpret_cast<long long*>(step), R, 0, st);
}

int lvsr_logprobs(lvsr_model* m, const float* attended, const float* preprocessed, const float* attended_mask,
                  int32_t Tp, int32_t U, const int32_t* row_utt, int32_t R, const float* states,
                  const float* weights, const int64_t* step, float* out, void* stream) {
  return lvsr_logprobs_lm(m, attended, preprocessed, attended_mask, Tp, U, row_utt, R, states, weights, step, nullptr,
                          out, stream);
}

int lvsr_logprobs_lm(lvsr_model* m, const float* attended, const float* preprocessed, const float* attended_mask,
                     int32_t Tp, int32_t U, const int32_t* row_utt, int32_t R, const float* states,
                     const float* weights, const int64_t* step, const float* lm_add, float* out, void* stream) {
  DeviceGuard device_guard(m);
  if (int rc = bind_stream(m, static_cast<cudaStream_t>(stream))) return rc;
  if (int rc = check_ready(m)) return rc;
  LVSR_CHECK(attended && attended_mask && states && weights && step && out && Tp > 0 && U > 0 && R > 0,
             "logprobs: bad arguments");
  LVSR_CHECK(row_utt || U == R, "logprobs: without row_utt the contexts must be replicated (U == R)");
  LVSR_CHECK(!lm_add || lm_attached(m), "logprobs: language-model cost rows given but no language model attached");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ArenaScope scope(m, st);
  const lvsr_config& c = m->cfg;
  Arena& ws = m->ws;
  const float* P = preprocessed;
  if (!P) {
    float* Pb = ws.f32((size_t)Tp * U * c.dim_matcher);
    LVSR_CHECK(Pb, "out of device memory (preprocessed)");
    if (int rc = lvsr_preprocess(m, attended, Tp, U, Pb, stream)) return rc;
    P = Pb;
  }
  float* w_tmp = ws.f32((size_t)R * Tp);
  float* e_tmp = ws.f32((size_t)R * Tp);
  float* ctx = ws.f32((size_t)R * m->E);
  float* merged = ws.f32((size_t)R * c.post_merge_dim);
  LVSR_CHECK(w_tmp && e_tmp && ctx && merged, "out of device memory (logprobs workspace)");
  if (int rc = glimpses(m, attended, P, attended_mask, Tp, U, row_utt, R, states, weights,
                        reinterpret_cast<const long long*>(step), 0, w_tmp, e_tmp, ctx, st)) return rc;
  const float* tail = nullptr;
  if (int rc = readout_merged(m, R, states, ctx, merged, &tail, st)) return rc;
  ReadoutArgs r = readout_args(m, R, tail);
  r.costs_all = out;
  if (lm_add) lm_fuse(m, r, lm_add);
  return readout_costs(r, st);
}

int lvsr_next_states(lvsr_model* m, const float* attended, const float* preprocessed, const float* attended_mask,
                     int32_t Tp, int32_t U, const int32_t* row_utt, int32_t R, const float* states,
                     const float* weights, const int64_t* step, const int64_t* outputs, float* next_states,
                     float* next_wavg, float* next_weights, float* next_energies, int64_t* next_step, void* stream) {
  DeviceGuard device_guard(m);
  if (int rc = bind_stream(m, static_cast<cudaStream_t>(stream))) return rc;
  if (int rc = check_ready(m)) return rc;
  LVSR_CHECK(attended && attended_mask && states && weights && step && outputs && next_states && next_wavg &&
                 next_weights && next_energies && next_step && Tp > 0 && U > 0 && R > 0,
             "next_states: bad arguments");
  LVSR_CHECK(row_utt || U == R, "next_states: without row_utt the contexts must be replicated (U == R)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ArenaScope scope(m, st);
  const lvsr_config& c = m->cfg;
  Arena& ws = m->ws;
  const float* P = preprocessed;
  if (!P) {
    float* Pb = ws.f32((size_t)Tp * U * c.dim_matcher);
    LVSR_CHECK(Pb, "out of device memory (preprocessed)");
    if (int rc = lvsr_preprocess(m, attended, Tp, U, Pb, stream)) return rc;
    P = Pb;
  }
  if (int rc = glimpses(m, attended, P, attended_mask, Tp, U, row_utt, R, states, weights,
                        reinterpret_cast<const long long*>(step), 0, next_weights, next_energies, next_wavg, st)) return rc;
  if (int rc = transition(m, R, states, next_wavg, reinterpret_cast<const long long*>(outputs), nullptr, next_states, st))
    return rc;
  return add_i64(reinterpret_cast<long long*>(next_step), reinterpret_cast<const long long*>(step), R, 1, st);
}

}  // extern "C"

namespace lvsr {

int search_expand(lvsr_model* m, const float* attended, const float* preprocessed, const float* attended_mask, int Tp,
                  int U, const int* utt_len, const int* row_utt, const int* row_seg, const int* seg_start, int nseg,
                  int R, const float* states, const float* weights, const long long* step, const float* cost_so_far,
                  const float* lm_add, int k, float* wavg, float* new_weights, float* new_energies, int* top_parent,
                  int* top_symbol, float* top_cost, int* top_count, cudaStream_t st) {
  ArenaScope scope(m, st);
  const lvsr_config& c = m->cfg;
  Arena& ws = m->ws;
  float* merged = ws.f32((size_t)R * c.post_merge_dim);
  float* neglogp = ws.f32((size_t)R * c.num_phonemes);
  LVSR_CHECK(merged && neglogp, "out of device memory (search workspace)");
  Segments sg;
  sg.seg_start = seg_start; sg.nseg = nseg; sg.seg_len = utt_len; sg.row_seg = row_seg;
  // take_glimpses ONCE per hypothesis: the same glimpse feeds the readout (logprobs_computer) and, for the
  // surviving parents, the state update (next_state_computer) -- B/search.py:109-142 computes it twice
  if (int rc = glimpses(m, attended, preprocessed, attended_mask, Tp, U, row_utt, R, states, weights, step, 0,
                        new_weights, new_energies, wavg, st, sg)) return rc;
  const float* tail = nullptr;
  if (int rc = readout_merged(m, R, states, wavg, merged, &tail, st)) return rc;
  ReadoutArgs r = readout_args(m, R, tail);
  r.costs_all = neglogp;
  if (lm_add) lm_fuse(m, r, lm_add);
  if (int rc = readout_costs(r, st)) return rc;
  return segment_topk(neglogp, cost_so_far, seg_start, nseg, c.num_phonemes, k, top_parent, top_symbol, top_cost, top_count, st);
}

int search_advance(lvsr_model* m, const float* attended, const float* preprocessed, const float* attended_mask, int Tp,
                   int U, const int* utt_len, int Rn, const int* parent, const long long* symbols, const int* row_utt,
                   const int* row_seg, const int* seg_start, int nseg, const float* states, const float* weights,
                   const long long* step, const float* wavg, const float* new_weights, const float* new_energies,
                   float* n_states, float* n_wavg, float* n_weights, float* n_energies, long long* n_step,
                   cudaStream_t st) {
  ArenaScope scope(m, st);
  const lvsr_config& c = m->cfg;
  Arena& ws = m->ws;
  const int S = state_dim(m), E = m->E;
  float* s_sel = ws.f32((size_t)Rn * S);
  LVSR_CHECK(s_sel, "out of device memory (search workspace)");
  if (int rc = gather_rows(s_sel, states, parent, Rn, S, st)) return rc;
  if (c.prior_type == LVSR_PRIOR_EXPANDING) {
    if (int rc = gather_rows(n_wavg, wavg, parent, Rn, E, st)) return rc;
    if (int rc = gather_rows(n_weights, new_weights, parent, Rn, Tp, st)) return rc;
    if (int rc = gather_rows(n_energies, new_energies, parent, Rn, Tp, st)) return rc;
  } else {
    // window priors: the reference recomputes the glimpses over the SELECTED parents, whose batch-global cut
    // (lvsr/bricks/attention.py:151-152) can differ from the cut over the whole beam
    float* w_sel = ws.f32((size_t)Rn * Tp);
    long long* st_sel = ws.i64((size_t)Rn);
    LVSR_CHECK(w_sel && st_sel, "out of device memory (search workspace)");
    if (int rc = gather_rows(w_sel, weights, parent, Rn, Tp, st)) return rc;
    if (int rc = gather_i64(st_sel, step, parent, Rn, 0, st)) return rc;
    Segments sg;
    sg.seg_start = seg_start; sg.nseg = nseg; sg.seg_len = utt_len; sg.row_seg = row_seg;
    if (int rc = glimpses(m, attended, preprocessed, attended_mask, Tp, U, row_utt, Rn, s_sel, w_sel, st_sel, 0, n_weights,
                          n_energies, n_wavg, st, sg)) return rc;
  }
  if (int rc = transition(m, Rn, s_sel, n_wavg, symbols, nullptr, n_states, st)) return rc;
  return gather_i64(n_step, step, parent, Rn, 1, st);
}

}  // namespace lvsr

extern "C" {

int lvsr_recognizer_cost_host(lvsr_model* m, const float* x_h, const float* mask_h, const int64_t* labels_h,
                              const float* lmask_h, int32_t T, int32_t B, int32_t L, float* costs_h, void* stream) {
  DeviceGuard device_guard(m);
  if (int rc = bind_stream(m, static_cast<cudaStream_t>(stream))) return rc;
  if (int rc = check_ready(m)) return rc;
  LVSR_CHECK(x_h && labels_h && costs_h && T > 0 && B > 0 && L > 0, "recognizer_cost_host: bad arguments");
  for (long long i = 0; i < (long long)L * B; ++i)       // host memory: the lookup's IndexError, up front
    LVSR_CHECK(labels_h[i] >= 0 && labels_h[i] < m->cfg.num_phonemes,
               "recognizer_cost_host: label %lld at [%lld, %lld] outside [0, %d)", (long long)labels_h[i], i / B, i % B,
               m->cfg.num_phonemes);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = 0;
  {
    const int F = m->cfg.num_features, Tp = lvsr_encoded_length(m, T), E = m->E;
    m->ws.reserve(encoder_ws_bytes(m, T, B) + cost_ws_bytes(m, Tp, B, L) +
                      ((size_t)T * B * (F + 1) + (size_t)3 * L * B + (size_t)Tp * B * (E + 1)) * sizeof(float) + (1 << 16),
                  st);
    ArenaScope scope(m, st);
    Arena& ws = m->ws;
    float* x = ws.f32((size_t)T * B * F);
    float* mask = mask_h ? ws.f32((size_t)T * B) : nullptr;
    long long* lab = ws.i64((size_t)L * B);
    float* lmask = lmask_h ? ws.f32((size_t)L * B) : nullptr;
    float* att = ws.f32((size_t)Tp * B * E);
    float* attm = ws.f32((size_t)Tp * B);
    float* costs = ws.f32((size_t)L * B);
    LVSR_CHECK(x && lab && att && attm && costs && (!mask_h || mask) && (!lmask_h || lmask), "out of device memory (host call)");
    LVSR_CUDA_OK(cudaMemcpyAsync(x, x_h, (size_t)T * B * F * sizeof(float), cudaMemcpyHostToDevice, st));
    if (mask) LVSR_CUDA_OK(cudaMemcpyAsync(mask, mask_h, (size_t)T * B * sizeof(float), cudaMemcpyHostToDevice, st));
    LVSR_CUDA_OK(cudaMemcpyAsync(lab, labels_h, (size_t)L * B * sizeof(long long), cudaMemcpyHostToDevice, st));
    if (lmask) LVSR_CUDA_OK(cudaMemcpyAsync(lmask, lmask_h, (size_t)L * B * sizeof(float), cudaMemcpyHostToDevice, st));
    rc = lvsr_encoder_forward(m, x, mask, T, B, att, attm, stream);
    if (!rc) rc = lvsr_cost_matrix(m, att, attm, Tp, B, reinterpret_cast<const int64_t*>(lab), lmask, L, costs,
                                   nullptr, nullptr, nullptr, nullptr, stream);
    if (!rc) {
      unsigned hst = 0;
      LVSR_CUDA_OK(cudaMemcpyAsync(costs_h, costs, (size_t)L * B * sizeof(float), cudaMemcpyDeviceToHost, st));
      LVSR_CUDA_OK(cudaMemcpyAsync(&hst, m->status.get(), sizeof(hst), cudaMemcpyDeviceToHost, st));
      LVSR_CUDA_OK(cudaStreamSynchronize(st));
      if (hst != 0) {
        // the persistent decoder gave up (status in common.cuh): same math on the step-wise kernels
        if (m->dec_fallbacks++ == 0)
          fprintf(stderr, "[lvsr_b200] persistent decoder launch failed (status %u); re-running on the step-wise kernels\n", hst);
        m->force_stepwise = true;
        rc = lvsr_cost_matrix(m, att, attm, Tp, B, reinterpret_cast<const int64_t*>(lab), lmask, L, costs,
                              nullptr, nullptr, nullptr, nullptr, stream);
        m->force_stepwise = false;
        if (!rc) {
          LVSR_CUDA_OK(cudaMemcpyAsync(costs_h, costs, (size_t)L * B * sizeof(float), cudaMemcpyDeviceToHost, st));
          LVSR_CUDA_OK(cudaStreamSynchronize(st));
        }
      }
    }
  }
  return rc;
}

}  // extern "C"
