// Training step of the recognizer: cost, gradients of every parameter, and the step rules.
//
// Replaces GradientDescent._function (libs/blocks/blocks/algorithms/__init__.py:244-256,284-287) built by
// lvsr/main.py:340-345,480-519: cost = sum(cost_matrix) / batch size, gradients by back-propagation
// through the decoder scan (attention + GRU), the readout and the pyramidal BiGRU encoder, then
// StepClipping -> Momentum -> AdaDelta -> Restrict(VariableClipping(axis=0), WEIGHT) -> RemoveNotFinite(0.0)
// -> BurnIn and the in-place update.  The gradient buffer uses the flat parameter layout, so a data-parallel
// caller all-reduces ONE buffer between lvsr_train_cost_and_grads and lvsr_train_apply_updates (SURVEY.md 8e).
//
// TrainStep::run: taped forward (DecTape), the transposed weights (made in run, ahead of the readout's buffers, for their
// place in the arena), readout backward, decoder backward (the reverse-time loop: DecGrads), decoder weight gradients,
// gradient of the attended sequence, encoder backward.  Work off the recurrences is LARGE GEMMs over all steps.  The
// recurrences are reverse-time scans: bigru_bwd.cu (persistent cluster kernel) and the decoder loop (per step: 4 skinny
// products, the attention backward re-computing tanh(match) instead of storing [L,T',B,M], two element-wise kernels).
#include <stdlib.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "model.h"
#include "train_kernels.cuh"

using namespace lvsr;
using namespace lvsr::train;

namespace {

inline int grid1d(long long n, int block = 256, int cap = 2048) {
  return (int)std::min<long long>(cap, std::max<long long>(1, (n + block - 1) / block));
}

// C[Mo,N] (ldc) (+)= A[:, m-cols]^T . B over R rows; *splits_out (may be null) = the partial products of the R rows
int gemm_tn(Arena& ws, const float* A, int lda, const float* B, int ldb, int R, int Mo, int N, float* C, int ldc,
            bool accumulate, cudaStream_t st, int* splits_out = nullptr) {
  ProfScope prof("gemm_tn", st);
  if (splits_out) *splits_out = 0;
  if (R <= 0 || Mo <= 0 || N <= 0) return 0;
  const int tiles = ceil_div(Mo, TN_BM) * ceil_div(N, TN_BN);
  int splits = std::max(1, std::min(ceil_div(2 * device_sm_count(), tiles), ceil_div(R, 4 * TN_BK)));
  int rps = ceil_div(ceil_div(R, splits), TN_BK) * TN_BK;
  splits = ceil_div(R, rps);
  if (splits_out) *splits_out = splits;
  ArenaMark mark{ws};                       // partials are dead once the reduce is enqueued (stream order)
  float* part = ws.f32((size_t)splits * Mo * N);
  LVSR_CHECK(part, "out of device memory (TN partials)");
  TnArgs g;
  g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.R = R; g.Mo = Mo; g.N = N; g.part = part; g.rows_per_split = rps;
  g.vec_a = lda % 4 == 0 && reinterpret_cast<uintptr_t>(A) % 16 == 0;
  g.vec_b = ldb % 4 == 0 && reinterpret_cast<uintptr_t>(B) % 16 == 0;
  dim3 grid(ceil_div(N, TN_BN), ceil_div(Mo, TN_BM), splits);
  gemm_tn_kernel<<<grid, 256, 0, st>>>(g);
  LVSR_LAUNCH_CHECK();
  tn_reduce_kernel<<<grid1d((long long)Mo * N), 256, 0, st>>>(part, splits, Mo, N, C, ldc, accumulate ? 1 : 0);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int gemm_nn(const float* A, int M, int K, int lda, const float* W, int N, int ldw, const float* bias, float* C, int ldc,
            bool accumulate, cudaStream_t st) {
  GemmArgs g = make_gemm(A, M, K, W, N, bias, C, accumulate);
  g.lda = lda; g.ldw = ldw; g.ldc = ldc;
  return gemm_bias(g, st);
}

int colsum(const float* X, int R, int N, int ldx, float* out, bool accumulate, cudaStream_t st) {
  if (N <= 0) return 0;
  colsum_kernel<<<ceil_div(N, 32), 256, 0, st>>>(X, R, N, ldx, out, accumulate ? 1 : 0);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int transpose(const float* src, float* dst, int K, int N, cudaStream_t st) {
  dim3 grid(ceil_div(N, 32), ceil_div(K, 32)), block(32, 8);
  transpose_kernel<<<grid, block, 0, st>>>(src, dst, K, N);
  LVSR_LAUNCH_CHECK();
  return 0;
}

int skinny(const float* X0, int K0, int ldx0, const float* W0, const float* X1, int K1, int ldx1, const float* W1,
           const float* add0, int lda0, const float* add1, int lda1, float* out, int ldo, int R, int N, cudaStream_t st,
           int split = 0, float* out1 = nullptr, int ldo1 = 0) {
  LVSR_CHECK(N % 4 == 0 && K0 % 4 == 0 && (X1 == nullptr || K1 % 4 == 0) && ldx0 % 4 == 0, "skinny: dimensions must be multiples of 4");
  SkinnyArgs a = {};
  a.X[0] = X0; a.K[0] = K0; a.ldx[0] = ldx0; a.W[0] = W0;
  a.X[1] = X1; a.K[1] = K1; a.ldx[1] = ldx1; a.W[1] = W1;
  a.add[0] = add0; a.lda[0] = lda0; a.add[1] = add1; a.lda[1] = lda1;
  a.out = out; a.ldo = ldo; a.R = R; a.N = N;
  a.split = split; a.out1 = out1; a.ldo1 = ldo1;
  LVSR_CHECK(split % SK_N == 0, "skinny: the column split must be a multiple of %d", SK_N);
  dim3 grid(ceil_div(N, SK_N), ceil_div(R, SK_R));
  ProfScope prof("skinny", st);
  skinny_kernel<<<grid, SK_WARPS * 32, 0, st>>>(a);
  LVSR_LAUNCH_CHECK();
  return 0;
}

// K-major (contraction-major) tf32 hi/lo operand of the tensor-core GEMM: [rows, Kpad] built from a [K, rows] matrix
struct TcOperand { float* hi = nullptr; float* lo = nullptr; int Kpad = 0; };

// src [R, cols] (leading dimension ld) -> transposed hi/lo pair [cols, kpad(R)]
int make_tc_operand(Arena& ws, const float* src, int R, int cols, int ld, TcOperand* out, cudaStream_t st) {
  out->Kpad = gemm_tc_kpad(R);
  out->hi = ws.f32((size_t)cols * out->Kpad);
  out->lo = ws.f32((size_t)cols * out->Kpad);
  LVSR_CHECK(out->hi && out->lo, "out of device memory (tensor-core operand)");
  return transpose_split_tf32(src, R, cols, ld, out->hi, out->lo, st);
}

// Rows of the contraction one split of gemm_tn_tc adds up in its tensor-core accumulators, at most, and the most splits
// the training step's arena holds partials for (TrainStep::run).  The error of a split grows with the rows it adds, far
// faster than that of an fp32 FFMA sum: on the benchmarked training batch (T * B = 96,000 rows) the fork weight
// gradients of encoder layers 1 and 2 were off by up to 1.4e-4 of their largest entry at 16,000 rows per split and by
// 4e-5 at 2048 (H100 SXM, 700 W).  The partials are summed in fp32.
constexpr int TC_SPLIT_ROWS = 2048, TC_MAX_SPLITS = 80;

// C[Mo, N] (ldc) (+)= A^T B on the tensor cores: A, B given as K-major operands (rows a0.. / b0..), split-K over the
// contraction (R) so that every SM gets a tile and no split adds more than TC_SPLIT_ROWS rows; partials are summed in a
// fixed order.  *splits_out (may be null) = the partial products launched.
int gemm_tn_tc(Arena& ws, const TcOperand& A, int a0, int Mo, const TcOperand& B, int b0, int N, float* C, int ldc,
               bool accumulate, cudaStream_t st, int* splits_out = nullptr) {
  ProfScope prof("gemm_tn", st);
  const int tiles = ceil_div(Mo, 128) * (N / (N % 256 == 0 ? 256 : 128));
  const int want = std::min(TC_MAX_SPLITS, std::max({1, std::min(32, ceil_div(device_sm_count(), tiles)),
                                                     ceil_div(A.Kpad, TC_SPLIT_ROWS)}));
  const int splits = gemm_tc_splits_launched(A.Kpad, want);
  if (splits_out) *splits_out = splits;
  ArenaMark mark{ws};
  float* part = ws.f32((size_t)splits * Mo * N);
  LVSR_CHECK(part, "out of device memory (TN partials)");
  if (int rc = gemm_tc_presplit(A.hi + (size_t)a0 * A.Kpad, A.lo + (size_t)a0 * A.Kpad, Mo, B.hi + (size_t)b0 * B.Kpad,
                                B.lo + (size_t)b0 * B.Kpad, N, A.Kpad, nullptr, part, N, want, (long long)Mo * N, st)) return rc;
  tn_reduce_kernel<<<grid1d((long long)Mo * N), 256, 0, st>>>(part, splits, Mo, N, C, ldc, accumulate ? 1 : 0);
  LVSR_LAUNCH_CHECK();
  return 0;
}

// The decoder's tape: attended sequence and mask, per step costs, alignments, energies (softmax: null), s_{i-1}, glimpses,
// and under a task-loss criterion what its loss was formed from (log-likelihood: null)
struct DecTape { float *Hatt, *attm, *costs, *W_all, *E_all, *S_prev, *CTX; TleTape tle; };
// Greedy exploration (lvsr/main.py:245-283): the step generates its own `labels` (prediction) and `lmask` (the
// prediction's mask) into these buffers after the encoder, and the task-loss rewards compare them with `groundtruth`
struct Greedy { const int64_t* groundtruth; int Lg; long long* prediction; float* prediction_mask; };
// Decoder backward's results: [dGz|dGr|dA], re-computed HR, dCTX, dq partials [L][2][B][M], dP, attention-constant partials
struct DecGrads { float *dG, *HR, *dCTX, *dQp, *dP, *acc_v, *acc_Wh, *acc_filt, *acc_b; };

// One training step's shapes and handles; phases read parameters via m->P as they run (adaptive noise re-points them)
struct TrainStep {
  lvsr_model* m;
  cudaStream_t st;
  const int64_t* labels;
  const float* lmask;
  float* grads;
  float gscale;
  int B, L, Tp;
  const DropoutKey* drop;          // dropout on the encoder's input (null: off)
  float penalty_coof;              // alignment penalty coefficient (0: off)
  const Greedy* greedy = nullptr;  // greedy exploration (null: the labels are the decoder's outputs)
  const lvsr_config& c = m->cfg;
  Arena& ws = m->tws;
  const long long* lab = reinterpret_cast<const long long*>(labels);
  const int C = c.dim_dec, E = m->E, M = c.dim_matcher, K = c.conv_num_filters, n = c.conv_n, w = 2 * n + 1;
  // Hd: the readout tail's hidden width, d_k / pieces (pieces is 1 above depth 1)
  const int V = c.num_phonemes, Cfb = c.dim_feedback, Cpm = c.post_merge_dim, Kro = readout_depth(m);
  const int Hd = readout_dim(m, Kro - 1) / c.maxout_pieces;
  const int R = L * B, nct = AB_CS * B, tc_cap = ceil_div(Tp, AB_CS);
  const bool content = content_attention(m);
  const bool tle = tle_criterion(m);
  // the logistic and relu energy gradients read the step's energies, which the softmax one does not need
  const bool keep_energies = c.energy_normalizer != LVSR_NORM_SOFTMAX;
  const size_t ro_smem = readout_bwd_smem_bytes(Hd);
  const size_t ab_smem = (content ? att_bwd_content_smem_floats(E, tc_cap) : att_bwd_smem_floats(M, E, K, n, tc_cap)) * sizeof(float);
  const std::string g = GEN, t = TR, at = att_base(m);
  float* grad(const std::string& name) const { const Param* p = m->param(name); return p ? grads + p->offset : nullptr; }

  int run(const float* x, const float* mask, int T, float* cost_out) const {
    // shapes the backward kernels cannot take are refused before any work is enqueued
    LVSR_CHECK(ro_smem <= READOUT_SMEM_LIMIT && V <= 128, "readout backward: post_merge_dim / num_phonemes too large");
    LVSR_CHECK(ab_smem <= 227 * 1024 && M <= AB_NT && M % 128 == 0 && K <= 16 && E % 4 == 0,
               "attention backward: shape unsupported (Tp=%d M=%d)", Tp, M);
    LVSR_CHECK(E <= 1024, "encoded dim %d > 1024 unsupported in training", E);
    // size the tape arena once per shape
    size_t bytes = (size_t)64 << 20;
    int Tl = T, din = encoder_input_dim(m);
    for (int i = 0; i < m->bottom.num_layers; ++i) {
      // output, forward split, K-major operands, TN partials and the input gradient with its operands
      const size_t rows = (size_t)T * B, di = bottom_input_dim(m, i), d = m->bottom.dims[i];
      bytes += (rows * d + 2 * rows * gemm_tc_kpad((int)di) + 2 * (di + d + 32) * (rows + 32) + (size_t)80 * di * d +
                rows * di + 2 * rows * d + 2 * di * d) * sizeof(float);
    }
    for (int l = 0; l < c.num_layers; ++l) {
      // N: the fork's columns (3 ndir D), Dout: the layer's output (ndir D)
      const int D = c.dims_bidir[l], Tout = ceil_div(Tl, c.subsample[l]), N = encoder_fork(m, l, 0).ld;
      const int Dout = encoder_output_dim(m, l);
      bytes += ((size_t)Tl * B * N * 2 + (size_t)(Tl + 2) * B * Dout * 2 + (size_t)Tout * B * Dout * 2 + (size_t)3 * Tl * B * gemm_tc_kpad(din)) * sizeof(float);
      bytes += (size_t)80 * std::max(din, Dout) * N * sizeof(float);      // TN partials
      bytes += ((size_t)2 * (N + din + 3 * D + 32) * (Tl * (size_t)B + 32) + (size_t)2 * Tl * B * N) * sizeof(float);   // K-major tf32 operands
      Tl = Tout; din = Dout;
    }
    bytes += ((size_t)Tp * B * (2 * M + 2 * E) + (size_t)R * (Tp + 8 * C + 3 * E + 2 * M + 3 * Cpm + V + 16) + (size_t)4 * B * Tp +
              (size_t)2 * B * (M + (size_t)K * M + (size_t)K * w) + (size_t)4 * (E + C) * 3 * C + (size_t)80 * E * M) * sizeof(float);
    if (keep_energies) bytes += ((size_t)R * Tp + (size_t)AB_CS * B) * sizeof(float);
    for (int j = 1; j < Kro; ++j)         // the readout body: h_j, dh_j, z's gradient, W_{j-1}^T and TN partials
      bytes += ((size_t)3 * R * readout_dim(m, j) + (size_t)81 * readout_dim(m, j - 1) * readout_dim(m, j) + 1024) * sizeof(float);
    if (drop) bytes += (size_t)T * B * encoder_input_dim(m) * sizeof(float);      // the dropped encoder input
    if (penalty_coof > 0.f) bytes += (size_t)R * (Tp + 1) * sizeof(float);      // penalty gradient and row sums
    if (tle) bytes += (size_t)3 * R * V * sizeof(float) + (size_t)R * sizeof(double);   // the loss's inputs, its row sums
    ws.reserve(bytes, st);
    ArenaScope scope(ws, st);
    for (int l = 0; l < c.num_layers; ++l)
      for (int s = LVSR_ENC_BWD_CS; s <= LVSR_ENC_DX; ++s) m->enc_plan[l][s] = 0;
    LVSR_CUDA_OK(cudaMemsetAsync(grads, 0, (size_t)m->flat_count * sizeof(float), st));
    std::vector<LayerTape> tape(c.num_layers);
    const float* bottom_out[LVSR_MAX_BOTTOM] = {};
    DecTape d;
    if (int rc = taped_forward(x, mask, T, tape.data(), bottom_out, cost_out, d)) return rc;
    // dY . W^T right-hand sides, transposed here, not in the phases that read them, to keep their arena place ahead of
    // the readout's and decoder backward's buffers: placement can move the step time (DESIGN.md section 6, item 4)
    float* WmsT = c.use_states_for_readout ? ws.f32((size_t)Cpm * C) : nullptr;     // [Cpm, C]
    float* WmcT = ws.f32((size_t)Cpm * E);
    float* WstateT = ws.f32((size_t)C * C);
    float* WgT = ws.f32((size_t)2 * C * C);             // [2C, C]
    float* WdcatT = ws.f32((size_t)3 * C * E);          // [3C, E]
    float* WsT = ws.f32((size_t)M * C);                 // [M, C]
    float* WpT = ws.f32((size_t)M * E);                 // [M, E]
    LVSR_CHECK(WmcT && WstateT && WgT && WdcatT && WsT && WpT, "out of device memory (transposed weights)");
    if (WmsT) if (int rc = transpose(m->P(g + "/readout/merge/transform_states.W"), WmsT, C, Cpm, st)) return rc;
    if (int rc = transpose(m->P(g + "/readout/merge/transform_weighted_averages.W"), WmcT, E, Cpm, st)) return rc;
    if (int rc = transpose(m->P(t + "/transition.state_to_state"), WstateT, C, C, st)) return rc;
    if (int rc = transpose(m->P(t + "/transition.state_to_gates"), WgT, C, 2 * C, st)) return rc;
    if (int rc = transpose(m->dec[0].Wd.get(), WdcatT, E, 3 * C, st)) return rc;
    // [dG (3C)] . WcombT [3C, C + E] = [ grad of s_{i-1} through the gates | grad of the glimpse ]: one product per step
    float* WcombT = ws.f32((size_t)3 * C * (C + E));
    LVSR_CHECK(WcombT, "out of device memory (transposed weights)");
    LVSR_CUDA_OK(cudaMemsetAsync(WcombT, 0, (size_t)3 * C * (C + E) * sizeof(float), st));
    if (int rc = copy2d(WcombT, C + E, WgT, C, 2 * C, C, st)) return rc;
    if (int rc = copy2d(WcombT + C, C + E, WdcatT, E, 3 * C, E, st)) return rc;
    if (int rc = transpose(m->P(at + "/state_trans/transform_states.W"), WsT, C, M, st)) return rc;
    if (int rc = transpose(m->P(at + "/preprocess.W"), WpT, E, M, st)) return rc;
    float *dS_ro, *dCtx_ro, *dH;
    DecGrads dg;
    if (int rc = readout_backward(d, WmsT, WmcT, dS_ro, dCtx_ro)) return rc;
    if (int rc = decoder_backward(d, WstateT, WcombT, WsT, dS_ro, dCtx_ro, dg)) return rc;
    if (int rc = decoder_weight_grads(d, dg)) return rc;
    if (int rc = attended_grad(d, dg, WpT, dH)) return rc;
    if (int rc = encoder_backward(tape.data(), mask, dH, x, bottom_out)) return rc;
    // the groundtruth's eos check of the task-loss rewards waits for the whole step, not for its forward alone
    return tle ? tle_check_status(m, st) : 0;
  }
  // Taped forward: the encoder keeping its tape, then the teacher-forced decoder; *cost_out = sum(costs) * gscale
  int taped_forward(const float* x, const float* mask, int T, LayerTape* tape, const float** bottom_out, float* cost_out,
                    DecTape& d) const {
    d.Hatt = ws.f32((size_t)Tp * B * E);                  // attended [Tp, B, E]
    d.attm = ws.f32((size_t)Tp * B);
    LVSR_CHECK(d.Hatt && d.attm, "out of device memory (encoder output)");
    if (int rc = run_encoder(m, ws, x, mask, T, B, d.Hatt, d.attm, tape, st, bottom_out, drop)) return rc;
    if (greedy)
      if (int rc = tle_generate_greedy(m, d.Hatt, d.attm, Tp, B, L, greedy->prediction, greedy->prediction_mask, st)) return rc;
    d.tle = {};
    if (tle) {
      d.tle = {ws.f32((size_t)R * V), ws.f32((size_t)R * V), ws.f32((size_t)R * V)};
      LVSR_CHECK(d.tle.neg && d.tle.rewards && d.tle.gains, "out of device memory (task-loss tape)");
    }
    d.costs = ws.f32((size_t)R);
    d.W_all = ws.f32((size_t)R * Tp);        // alignments alpha_i
    d.S_prev = ws.f32((size_t)R * C);        // s_{i-1}
    d.CTX = ws.f32((size_t)R * E);           // weighted averages
    d.E_all = keep_energies ? ws.f32((size_t)R * Tp) : nullptr;     // energies e_i, bias included
    LVSR_CHECK(d.costs && d.W_all && d.S_prev && d.CTX && (d.E_all || !keep_energies), "out of device memory (decoder tape)");
    if (int rc = cost_matrix(m, d.Hatt, d.attm, Tp, B, labels, lmask, L, greedy ? greedy->groundtruth : nullptr,
                             greedy ? greedy->Lg : 0, d.costs, d.W_all, d.E_all, d.S_prev, d.CTX, tle ? &d.tle : nullptr, st))
      return rc;
    sum_all_kernel<<<1, 1024, 0, st>>>(d.costs, R, cost_out, gscale);
    LVSR_LAUNCH_CHECK();
    return 0;
  }
  // Readout + emitter backward, all steps at once; dS_ro / dCtx_ro: its gradients of the states and the glimpses.  Above
  // depth 1 the merge's epilogue makes h_0, the body the hidden layers up to the tail's input, and after the tail's
  // backward the body is walked top-down to the gradient of the merge.
  int readout_backward(const DecTape& d, const float* WmsT, const float* WmcT, float*& dS_ro, float*& dCtx_ro) const {
    const int Clast = readout_dim(m, Kro - 1);
    float* merged = ws.f32((size_t)R * Cpm);
    float* hid = ws.f32((size_t)R * Hd);
    float* dlogits = ws.f32((size_t)R * V);
    float* dmerged = ws.f32((size_t)R * Clast);
    dS_ro = ws.f32((size_t)R * C);
    dCtx_ro = ws.f32((size_t)R * E);
    LVSR_CHECK(merged && hid && dlogits && dmerged && dS_ro && dCtx_ro, "out of device memory (readout backward)");
    if (c.use_states_for_readout)
      if (int rc = gemm_nn(d.S_prev, R, C, C, m->P(g + "/readout/merge/transform_states.W"), Cpm, Cpm, nullptr, merged, Cpm, false, st)) return rc;
    {
      GemmArgs mc = make_gemm(d.CTX, R, E, m->P(g + "/readout/merge/transform_weighted_averages.W"), Cpm, nullptr, merged,
                              c.use_states_for_readout);
      if (Kro > 1) {
        mc.bias = m->P(g + "/readout/post_merge/bias.b");
        mc.act = c.post_merge_activation;
      }
      if (int rc = gemm_bias(mc, st)) return rc;
    }
    const float* h[LVSR_MAX_READOUT] = {};
    const float* tail = nullptr;
    if (int rc = readout_body(m, ws, R, merged, true, &tail, h, st)) return rc;
    const std::string top = readout_linear(Kro - 1);
    ReadoutBwdArgs rb = {};
    rb.merged = tail; rb.b_pm = m->P(Kro == 1 ? g + "/readout/post_merge/bias.b" : readout_linear(Kro - 2) + ".b");
    rb.Wo = m->P(top + ".W"); rb.bo = m->P(top + ".b");
    rb.R = R; rb.Cpm = Clast; rb.pieces = c.maxout_pieces; rb.V = V; rb.act = c.post_merge_activation;
    rb.labels = lab; rb.lmask = lmask; rb.gscale = gscale; rb.hid = hid; rb.dlogits = dlogits; rb.dmerged = dmerged;
    if (tle) {
      // RewardRegressionEmitter.cost's gradient (lvsr/bricks/__init__.py:135-184) in place of the softmax one
      double* row_sum = reinterpret_cast<double*>(ws.f32((size_t)2 * R));
      LVSR_CHECK(row_sum, "out of device memory (task-loss gradient)");
      const int loss = m->criterion.name == LVSR_CRITERION_MSE_GAIN ? LVSR_TLE_GAIN : LVSR_TLE_REWARD;
      if (int rc = tle_loss_grad(loss, d.tle.neg, d.tle.rewards, d.tle.gains, lab, lmask, L, B, V,
                                 (float)m->criterion.min_reward, gscale, row_sum, dlogits, st)) return rc;
      readout_bwd_kernel<true><<<ceil_div(R, 8), 256, ro_smem, st>>>(rb);
    } else {
      readout_bwd_kernel<false><<<ceil_div(R, 8), 256, ro_smem, st>>>(rb);
    }
    LVSR_LAUNCH_CHECK();
    if (int rc = gemm_tn(ws, hid, Hd, dlogits, V, R, Hd, V, grad(top + ".W"), V, false, st)) return rc;
    if (int rc = colsum(dlogits, R, V, V, grad(top + ".b"), false, st)) return rc;
    // dz: the gradient of the pre-activation of h_j, from j = k-1 down to 0 (h_0's is the merge's, dmerged [R, Cpm])
    float* dz = dmerged;
    for (int j = Kro - 2; j >= 0; --j) {
      ProfScope prof("readout_body_bwd", st);
      const int din = readout_dim(m, j), dout = readout_dim(m, j + 1);
      const std::string lin = readout_linear(j);
      if (int rc = colsum(dz, R, dout, dout, grad(lin + ".b"), false, st)) return rc;
      if (int rc = gemm_tn(ws, h[j], din, dz, dout, R, din, dout, grad(lin + ".W"), dout, false, st)) return rc;
      float* WT = ws.f32((size_t)dout * din);
      float* dh = ws.f32((size_t)R * din);
      LVSR_CHECK(WT && dh, "out of device memory (readout body backward)");
      if (int rc = transpose(m->P(lin + ".W"), WT, din, dout, st)) return rc;
      if (int rc = gemm_nn(dz, R, dout, dout, WT, din, din, nullptr, dh, din, false, st)) return rc;
      // Rectifier and Tanh from the stored output; Identity and Maxout(1) pass the gradient as it is
      if (c.post_merge_activation == LVSR_ACT_RELU || c.post_merge_activation == LVSR_ACT_TANH)
        if (int rc = bottom_act_backward(dh, h[j], (long long)R * din, c.post_merge_activation, st)) return rc;
      dz = dh;
    }
    dmerged = dz;
    if (int rc = colsum(dmerged, R, Cpm, Cpm, grad(g + "/readout/post_merge/bias.b"), false, st)) return rc;
    if (int rc = gemm_tn(ws, d.CTX, E, dmerged, Cpm, R, E, Cpm, grad(g + "/readout/merge/transform_weighted_averages.W"), Cpm, false, st)) return rc;
    if (int rc = gemm_nn(dmerged, R, Cpm, Cpm, WmcT, E, E, nullptr, dCtx_ro, E, false, st)) return rc;
    if (c.use_states_for_readout) {
      if (int rc = gemm_tn(ws, d.S_prev, C, dmerged, Cpm, R, C, Cpm, grad(g + "/readout/merge/transform_states.W"), Cpm, false, st)) return rc;
      if (int rc = gemm_nn(dmerged, R, Cpm, Cpm, WmsT, C, C, nullptr, dS_ro, C, false, st)) return rc;
    } else {
      LVSR_CUDA_OK(cudaMemsetAsync(dS_ro, 0, (size_t)R * C * sizeof(float), st));
    }
    return 0;
  }
  // Decoder backward: gate values of all steps re-computed, then the reverse-time loop; writes the initial state's gradient
  int decoder_backward(const DecTape& d, const float* WstateT, const float* WcombT, const float* WsT, const float* dS_ro,
                       const float* dCtx_ro, DecGrads& out) const {
    float* G = ws.f32((size_t)R * 3 * C);          // pre-activations -> third block keeps the candidate input
    float* Z = ws.f32((size_t)R * C);
    float* Rg = ws.f32((size_t)R * C);
    float* HR = ws.f32((size_t)R * C);
    float* Cc = ws.f32((size_t)R * C);
    float* Q = ws.f32((size_t)R * M);
    float* P = ws.f32((size_t)Tp * B * M);
    float* dP = ws.f32((size_t)Tp * B * M);
    float* dG = ws.f32((size_t)R * 3 * C);         // [dGz | dGr | dA] of every step
    float* dCTX = ws.f32((size_t)R * E);
    float* dQp = ws.f32((size_t)2 * R * M);        // the two CTAs' partial dq of every step
    float* dsbuf[2] = {ws.f32((size_t)B * C), ws.f32((size_t)B * C)};
    float* keep = ws.f32((size_t)B * C);
    float* dHR = ws.f32((size_t)B * C);
    float* dspart = ws.f32((size_t)B * C);
    float* dAbuf[2] = {ws.f32((size_t)2 * B * Tp), ws.f32((size_t)2 * B * Tp)};
    float* w0 = ws.f32((size_t)B * Tp);
    float* acc_v = ws.f32((size_t)nct * M);
    float* acc_Wh = ws.f32((size_t)nct * K * M);
    float* acc_filt = ws.f32((size_t)nct * K * w);
    float* acc_b = keep_energies ? ws.f32((size_t)nct) : nullptr;
    int* win = ws.i32(2);
    float* lohi = ws.f32((size_t)2 * B);
    LVSR_CHECK(G && Z && Rg && HR && Cc && Q && P && dP && dG && dCTX && dQp && dsbuf[0] && dsbuf[1] && keep && dHR && dspart &&
                   dAbuf[0] && dAbuf[1] && w0 && acc_v && (content || (acc_Wh && acc_filt)) && (acc_b || !keep_energies) &&
                   win && lohi,
               "out of device memory (decoder backward)");
    if (int rc = lvsr_preprocess(m, d.Hatt, Tp, B, P, st)) return rc;
    if (int rc = gemm_nn(d.CTX, R, E, E, m->dec[0].Wd.get(), 3 * C, 3 * C, nullptr, G, 3 * C, false, st)) return rc;
    if (int rc = gemm_nn(d.S_prev, R, C, C, m->P(t + "/transition.state_to_gates"), 2 * C, 2 * C, nullptr, G, 3 * C, true, st)) return rc;
    dec_gates_kernel<<<grid1d((long long)R * 3 * C), 256, 0, st>>>(G, m->dec[0].FF.get(), lab, d.S_prev, R, C, Z, Rg, HR);
    LVSR_LAUNCH_CHECK();
    {
      ArenaMark mark{ws};
      float* Cpre = ws.f32((size_t)R * C);
      LVSR_CHECK(Cpre, "out of device memory");
      if (int rc = gemm_nn(HR, R, C, C, m->P(t + "/transition.state_to_state"), C, C, nullptr, Cpre, C, false, st)) return rc;
      dec_cand_kernel<<<grid1d((long long)R * C), 256, 0, st>>>(Cpre, G, R, C, Cc);
      LVSR_LAUNCH_CHECK();
    }
    if (int rc = gemm_nn(d.S_prev, R, C, C, m->P(at + "/state_trans/transform_states.W"), M, M, nullptr, Q, M, false, st)) return rc;
    LVSR_CUDA_OK(cudaMemsetAsync(dP, 0, (size_t)Tp * B * M * sizeof(float), st));
    LVSR_CUDA_OK(cudaMemsetAsync(acc_v, 0, (size_t)nct * M * sizeof(float), st));
    if (!content) {
      LVSR_CUDA_OK(cudaMemsetAsync(acc_Wh, 0, (size_t)nct * K * M * sizeof(float), st));
      LVSR_CUDA_OK(cudaMemsetAsync(acc_filt, 0, (size_t)nct * K * w * sizeof(float), st));
    }
    if (acc_b) LVSR_CUDA_OK(cudaMemsetAsync(acc_b, 0, (size_t)nct * sizeof(float), st));
    LVSR_CUDA_OK(cudaMemsetAsync(dsbuf[0], 0, (size_t)B * C * sizeof(float), st));
    if (int rc = onehot_rows(w0, B, Tp, st)) return rc;
    // the alignment penalty's gradient of every alpha_i (it reads only the taped alignments) and its sum
    float* pen = nullptr;
    if (penalty_coof > 0.f) {
      ProfScope prof_pen("penalty", st);
      pen = ws.f32((size_t)R * Tp);
      float* rows = ws.f32((size_t)R);
      LVSR_CHECK(pen && rows, "out of device memory (alignment penalty)");
      penalty_grad_kernel<<<ceil_div(R, 256), 256, 0, st>>>(d.W_all, lmask, L, B, Tp, penalty_coof * gscale, pen, rows);
      LVSR_LAUNCH_CHECK();
      sum_all_kernel<<<1, 1024, 0, st>>>(rows, R, m->reg.penalty.get(), 1.f);
      LVSR_LAUNCH_CHECK();
    }
    void (*att_bwd)(AttBwdArgs, int) = att_bwd_content_kernel;
    if (!content) {
      const bool kp12 = att_bwd_kp(K) == 12;
      if (c.energy_normalizer == LVSR_NORM_LOGISTIC) att_bwd = kp12 ? att_bwd_kernel<12, LVSR_NORM_LOGISTIC> : att_bwd_kernel<16, LVSR_NORM_LOGISTIC>;
      else if (c.energy_normalizer == LVSR_NORM_RELU) att_bwd = kp12 ? att_bwd_kernel<12, LVSR_NORM_RELU> : att_bwd_kernel<16, LVSR_NORM_RELU>;
      else att_bwd = kp12 ? att_bwd_kernel<12, LVSR_NORM_SOFTMAX> : att_bwd_kernel<16, LVSR_NORM_SOFTMAX>;
    }
    LVSR_CUDA_OK(cudaFuncSetAttribute(att_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ab_smem));
    const int ew = ceil_div(B * C, 256);
    for (int i = L - 1; i >= 0; --i) {
      ProfScope prof("dec_bwd_step", st);
      const float* ds = dsbuf[(L - 1 - i) & 1];
      float* ds_next = dsbuf[(L - i) & 1];
      const float* lm_i = lmask ? lmask + (size_t)i * B : nullptr;
      float* dG_i = dG + (size_t)i * B * 3 * C;
      const float* Sp_i = d.S_prev + (size_t)i * B * C;
      dec_bwd_a_kernel<<<ew, 256, 0, st>>>(ds, Z + (size_t)i * B * C, Cc + (size_t)i * B * C, Sp_i, lm_i, B, C, dG_i, keep);
      LVSR_LAUNCH_CHECK();
      if (int rc = skinny(dG_i + 2 * C, C, 3 * C, WstateT, nullptr, 0, 0, nullptr, nullptr, 0, nullptr, 0, dHR, C, B, C, st)) return rc;
      dec_bwd_b_kernel<<<ew, 256, 0, st>>>(dHR, Rg + (size_t)i * B * C, Sp_i, B, C, dG_i, keep);
      LVSR_LAUNCH_CHECK();
      // grad of s_{i-1} through the gates (+ the element-wise paths), grad of the glimpse
      float* dctx_i = dCTX + (size_t)i * B * E;
      if (int rc = skinny(dG_i, 3 * C, 3 * C, WcombT, nullptr, 0, 0, nullptr, keep, C, dCtx_ro + (size_t)i * B * E, E, dspart, C, B, C + E, st,
                          C, dctx_i, E)) return rc;
      // attention backward
      const float* w_prev = i == 0 ? w0 : d.W_all + (size_t)(i - 1) * B * Tp;
      if (!content) {                     // content attention attends every frame: no window
        WindowArgs wa = {};
        wa.weights = w_prev; wa.step = nullptr; wa.step_offset = i; wa.R = B; wa.Tp = Tp; wa.prior = prior_of(c); wa.win = win; wa.lohi = lohi;
        if (int rc = attention_window(wa, st)) return rc;
      }
      AttBwdArgs ab = {};
      ab.P = P; ab.H = d.Hatt; ab.maskH = d.attm; ab.q = Q + (size_t)i * B * M; ab.w_prev = w_prev; ab.w_cur = d.W_all + (size_t)i * B * Tp;
      ab.ctx = d.CTX + (size_t)i * B * E; ab.dctx = dctx_i;
      ab.dA_in = (i == L - 1) ? nullptr : dAbuf[(L - 1 - i) & 1];
      ab.win = win;
      ab.filt = m->P(at + "/conv1d.filters"); ab.Wh = m->P(at + "/handler.W"); ab.v = m->P(at + "/energy_comp/linear.W");
      ab.dP = dP; ab.dq_part = dQp + (size_t)i * 2 * B * M; ab.dA_out = dAbuf[(L - i) & 1];
      ab.acc_v = acc_v; ab.acc_Wh = acc_Wh; ab.acc_filt = acc_filt;
      ab.B = B; ab.Tp = Tp; ab.M = M; ab.E = E; ab.K = K; ab.n = n;
      ab.e_cur = d.E_all ? d.E_all + (size_t)i * B * Tp : nullptr; ab.acc_b = acc_b;
      ab.pen = pen ? pen + (size_t)i * B * Tp : nullptr;
      {
        ProfScope prof_ab("att_bwd", st);
        att_bwd<<<nct, AB_NT, ab_smem, st>>>(ab, tc_cap);
        LVSR_LAUNCH_CHECK();
      }
      // ds_{i-1} = gates/elementwise part + dq . W_s^T (two partials) + readout of step i (which saw s_{i-1})
      const float* q0 = dQp + (size_t)i * 2 * B * M;
      if (int rc = skinny(q0, M, M, WsT, q0 + (size_t)B * M, M, M, WsT, dspart, C, dS_ro + (size_t)i * B * C, C, ds_next, C, B, C, st)) return rc;
    }
    // dsbuf[L & 1]: gradient of the broadcast initial state, per row
    if (int rc = colsum(dsbuf[L & 1], B, C, C, grad(t + "/transition.initial_state"), false, st)) return rc;
    out = {dG, HR, dCTX, dQp, dP, acc_v, acc_Wh, acc_filt, acc_b};
    return 0;
  }
  // Decoder weight gradients: large GEMMs over all steps, the feedback fork, and the sums of the attention constants
  int decoder_weight_grads(const DecTape& d, const DecGrads& dg) const {
    // state_to_state = HR^T dA ; state_to_gates = S_prev^T [dGz|dGr] ; distribute = CTX^T dG (gate columns first in dec[0].Wd)
    if (int rc = gemm_tn(ws, dg.HR, C, dg.dG + 2 * C, 3 * C, R, C, C, grad(t + "/transition.state_to_state"), C, false, st)) return rc;
    if (int rc = gemm_tn(ws, d.S_prev, C, dg.dG, 3 * C, R, C, 2 * C, grad(t + "/transition.state_to_gates"), 2 * C, false, st)) return rc;
    if (int rc = gemm_tn(ws, d.CTX, E, dg.dG, 3 * C, R, E, 2 * C, grad(t + "/distribute/fork_gate_inputs.W"), 2 * C, false, st)) return rc;
    if (int rc = gemm_tn(ws, d.CTX, E, dg.dG + 2 * C, 3 * C, R, E, C, grad(t + "/distribute/fork_inputs.W"), C, false, st)) return rc;
    // state transformer: S_prev^T dQ (two partials)
    {
      // dQp is [L][2][B][M]: view partial p as rows of length M with stride 2*B*M per step -> gather into [R, M] first
      ArenaMark mark{ws};
      float* dQ = ws.f32((size_t)R * M);
      LVSR_CHECK(dQ, "out of device memory");
      for (int p = 0; p < 2; ++p) {
        // rows of step i live at dQp + (i*2 + p)*B*M: a 2-D copy with pitch 2*B*M
        if (int rc = copy2d(dQ, B * M, dg.dQp + (size_t)p * B * M, 2 * B * M, L, B * M, st)) return rc;
        if (int rc = gemm_tn(ws, d.S_prev, C, dQ, M, R, C, M, grad(at + "/state_trans/transform_states.W"), M, p == 1, st)) return rc;
      }
    }
    // fork(feedback(y)): dFF by label, then lookup / fork weights / biases; the scratch is rewound when the phase returns
    ArenaMark mark{ws};
    float* dFF = ws.f32((size_t)(V + 1) * 3 * C);
    float* WffT = ws.f32((size_t)3 * C * Cfb);
    float* dWff = ws.f32((size_t)Cfb * 3 * C);
    float* dbff = ws.f32((size_t)3 * C);
    LVSR_CHECK(dFF && WffT && dWff && dbff, "out of device memory (feedback gradients)");
    scatter_rows_kernel<<<V + 1, 256, 0, st>>>(dg.dG, lab, R, 3 * C, dFF);
    LVSR_LAUNCH_CHECK();
    if (c.one_of_n_feedback) {
      // FF[y] = W_fork[y, :] + b: the gradient of the fork weights IS dFF
      LVSR_CUDA_OK(cudaMemcpyAsync(dWff, dFF, (size_t)(V + 1) * 3 * C * sizeof(float), cudaMemcpyDeviceToDevice, st));
    } else {
      if (int rc = transpose(m->dec[0].Wff.get(), WffT, Cfb, 3 * C, st)) return rc;
      const float* look = m->P(g + "/readout/lookupfeedback/lookuptable.W");
      if (int rc = gemm_nn(dFF, V + 1, 3 * C, 3 * C, WffT, Cfb, Cfb, nullptr, grad(g + "/readout/lookupfeedback/lookuptable.W"), Cfb, false, st)) return rc;
      if (int rc = gemm_tn(ws, look, Cfb, dFF, 3 * C, V + 1, Cfb, 3 * C, dWff, 3 * C, false, st)) return rc;
    }
    if (int rc = colsum(dFF, V + 1, 3 * C, 3 * C, dbff, false, st)) return rc;
    if (int rc = fork_copy(m, feedback_fork(c, 0), dWff, dbff, grads, st)) return rc;
    // attention constants: sums of the per-CTA partials
    reduce_partials_kernel<<<grid1d(M), 256, 0, st>>>(dg.acc_v, nct, M, grad(at + "/energy_comp/linear.W"));
    LVSR_LAUNCH_CHECK();
    if (!content) {
      reduce_partials_kernel<<<grid1d((long long)K * M), 256, 0, st>>>(dg.acc_Wh, nct, (long long)K * M, grad(at + "/handler.W"));
      LVSR_LAUNCH_CHECK();
      reduce_partials_kernel<<<grid1d((long long)K * w), 256, 0, st>>>(dg.acc_filt, nct, (long long)K * w, grad(at + "/conv1d.filters"));
      LVSR_LAUNCH_CHECK();
    }
    if (dg.acc_b) {
      reduce_partials_kernel<<<1, 256, 0, st>>>(dg.acc_b, nct, 1, grad(at + "/energy_comp/linear.b"));
      LVSR_LAUNCH_CHECK();
    }
    return 0;
  }
  // Gradient of the attended sequence (dH) through the glimpses and the preprocess, with the preprocess's gradients
  int attended_grad(const DecTape& d, const DecGrads& dg, const float* WpT, float*& dH) const {
    dH = ws.f32((size_t)Tp * B * E);
    LVSR_CHECK(dH, "out of device memory (dH)");
    dim3 grid(ceil_div(Tp, 8), B);
    dh_from_ctx_kernel<<<grid, 256, 0, st>>>(d.W_all, dg.dCTX, L, B, Tp, E, dH, 0);
    LVSR_LAUNCH_CHECK();
    if (int rc = gemm_nn(dg.dP, Tp * B, M, M, WpT, E, E, nullptr, dH, E, true, st)) return rc;
    if (int rc = gemm_tn(ws, d.Hatt, E, dg.dP, M, Tp * B, E, M, grad(at + "/preprocess.W"), M, false, st)) return rc;
    if (int rc = colsum(dg.dP, Tp * B, M, M, grad(at + "/preprocess.b"), false, st)) return rc;
    return 0;
  }
  // dX [rows, N] = dY [rows, K] . W^T for a layer's weights W [N, K] (row-major, so W is the K-major form of the
  // right-hand side): on the tensor cores when the shape suits them, else W transposed onto the FFMA tiles
  int input_grad(const float* dY, int rows, int K, const float* W, int N, float* dX, int32_t* path) const {
    if (m->use_tc && gemm_tc_supported(rows, N, K) && K % 32 == 0) {
      ArenaMark mark{ws};
      float* a_hi = ws.f32((size_t)rows * K);
      float* a_lo = ws.f32((size_t)rows * K);
      float* w_hi = ws.f32((size_t)N * K);
      float* w_lo = ws.f32((size_t)N * K);
      LVSR_CHECK(a_hi && a_lo && w_hi && w_lo, "out of device memory (dX operands)");
      if (int rc = split_tf32(W, w_hi, w_lo, (long long)N * K, st)) return rc;
      if (int rc = gemm_tc(dY, a_hi, a_lo, rows, K, w_hi, w_lo, N, nullptr, dX, N, st)) return rc;
      *path = LVSR_ENC_PATH_TC;
    } else {
      float* WT = ws.f32((size_t)K * N);
      LVSR_CHECK(WT, "out of device memory (dX)");
      if (int rc = transpose(W, WT, N, K, st)) return rc;
      if (int rc = gemm_nn(dY, rows, K, K, WT, N, N, nullptr, dX, N, false, st)) return rc;
      *path = LVSR_ENC_PATH_FFMA;
    }
    return 0;
  }
  // The bottom MLP, top layer first, from dY = the gradient of its output (overwritten): dZ = dY * act'(Y) in place,
  // dW_i = X_i^T dZ on the products of the fork weights, db_i = colsum(dZ), and dX_i = dZ W_i^T below the top layer.
  // Padded frames carry exactly zero dY (the BiGRU backward gives them no dPre), so they add nothing.
  int bottom_backward(const float* x, const float* const* Y, float* dY, int rows) const {
    ProfScope prof("bottom_bwd", st);
    const lvsr_bottom_config& bt = m->bottom;
    for (int i = bt.num_layers - 1; i >= 0; --i) {
      const int din = bottom_input_dim(m, i), d = bt.dims[i];
      const float* X = i ? Y[i - 1] : x;
      const std::string lin = bottom_linear(i);
      if (int rc = bottom_act_backward(dY, Y[i], (long long)rows * d, bt.activation, st)) return rc;
      {
        ArenaMark mark{ws};
        if (m->use_tc && rows >= 2048 && d % 128 == 0) {
          TcOperand dZT, XT;
          if (int rc = make_tc_operand(ws, dY, rows, d, d, &dZT, st)) return rc;
          if (int rc = make_tc_operand(ws, X, rows, din, din, &XT, st)) return rc;
          if (int rc = gemm_tn_tc(ws, XT, 0, din, dZT, 0, d, grad(lin + ".W"), d, false, st)) return rc;
        } else {
          if (int rc = gemm_tn(ws, X, din, dY, d, rows, din, d, grad(lin + ".W"), d, false, st)) return rc;
        }
      }
      if (int rc = colsum(dY, rows, d, d, grad(lin + ".b"), false, st)) return rc;
      if (i > 0) {
        float* dX = ws.f32((size_t)rows * din);
        LVSR_CHECK(dX, "out of device memory (bottom dX)");
        int32_t path = 0;
        if (int rc = input_grad(dY, rows, d, m->P(lin + ".W"), din, dX, &path)) return rc;
        dY = dX;
      }
    }
    return 0;
  }
  // Encoder backward, top layer first: scan, weight and input gradients; plan slots LVSR_ENC_BWD_CS .. LVSR_ENC_DX.
  // With a bottom MLP, layer 0's input gradient feeds its backward (x: the recordings, bottom_out: its layers' outputs).
  int encoder_backward(const LayerTape* tape, const float* mask, const float* dH, const float* x,
                       const float* const* bottom_out) const {
    const float* dout = dH;
    float* dX0 = nullptr;
    for (int l = c.num_layers - 1; l >= 0; --l) {
      const LayerTape& tp = tape[l];
      // nd directions side by side: the tape's rows are N = 3 nd D wide, hext's and hr's Dout = nd D
      const int D = tp.D, rows = tp.T * B, nd = encoder_dirs(m), N = 3 * nd * D, Dout = nd * D;
      float* hr = ws.f32((size_t)rows * Dout);
      float* dh0 = ws.f32((size_t)nd * B * D);
      LVSR_CHECK(hr && dh0, "out of device memory (encoder backward)");
      BiGruBwdArgs a = {};
      a.tape = tp.pre; a.hext = tp.hext; a.mask = mask; a.mask_tstride = tp.mstride; a.dout = dout;
      const std::string bf = enc_base(m, l, 0), bb = enc_base(m, l, 1);
      a.Wg_f = m->P(bf + "/gatedrecurrent.state_to_gates"); a.Ws_f = m->P(bf + "/gatedrecurrent.state_to_state");
      if (nd == 2) {
        a.Wg_b = m->P(bb + "/gatedrecurrent.state_to_gates"); a.Ws_b = m->P(bb + "/gatedrecurrent.state_to_state");
      }
      a.hr_out = hr; a.dh0 = dh0; a.T = tp.T; a.B = B; a.D = D; a.subsample = tp.k; a.ndir = nd;
      int32_t* plan = m->enc_plan[l];
      int bwd_cs = 0, wsplits = 0;
      if (int rc = bigru_layer_backward(a, st, &bwd_cs)) return rc;
      plan[LVSR_ENC_BWD_CS] = bwd_cs;
      // fork: dWcat = X^T dPre, dbcat = colsum(dPre), scattered to the parameters by the layer's fork layout
      {
        ArenaMark mark{ws};
        float* dWcat = ws.f32((size_t)tp.Din * N);
        float* dbcat = ws.f32((size_t)N);
        LVSR_CHECK(dWcat && dbcat, "out of device memory (fork gradients)");
        // tensor-core path: every operand transposed once into K-major tf32 hi/lo pairs (the contraction runs over the
        // T*B rows), then five split-K tensor-core products share them; FFMA tiles for small problems / LVSR_NO_TC_GEMM
        const bool tc = m->use_tc && rows >= 2048 && D % 128 == 0;
        // H_prev of each direction: slot t (forward) / t+2 (backward) of hext
        const float* hprev[2] = {tp.hext, tp.hext + (size_t)2 * B * Dout + D};
        TcOperand dPreT, XT, hrT, hpT[2];
        if (tc) {
          if (int rc = make_tc_operand(ws, tp.pre, rows, N, N, &dPreT, st)) return rc;
          if (int rc = make_tc_operand(ws, tp.X, rows, tp.Din, tp.Din, &XT, st)) return rc;
          if (int rc = make_tc_operand(ws, hr, rows, Dout, Dout, &hrT, st)) return rc;
          for (int dir = 0; dir < nd; ++dir)
            if (int rc = make_tc_operand(ws, hprev[dir], rows, D, Dout, &hpT[dir], st)) return rc;
          if (int rc = gemm_tn_tc(ws, XT, 0, tp.Din, dPreT, 0, N, dWcat, N, false, st, &wsplits)) return rc;
        } else {
          if (int rc = gemm_tn(ws, tp.X, tp.Din, tp.pre, N, rows, tp.Din, N, dWcat, N, false, st, &wsplits)) return rc;
        }
        plan[LVSR_ENC_WGRAD] = tc ? LVSR_ENC_PATH_TC : LVSR_ENC_PATH_FFMA;
        plan[LVSR_ENC_WGRAD_SPLITS] = wsplits;
        plan[LVSR_ENC_WGRAD_KPAD] = tc ? dPreT.Kpad : 0;
        if (int rc = colsum(tp.pre, rows, N, N, dbcat, false, st)) return rc;
        for (int dir = 0; dir < nd; ++dir) {
          const std::string b = enc_base(m, l, dir);
          const ForkLayout f = encoder_fork(m, l, dir);
          const int cA = f.block[0].col, cG = f.block[1].col;      // columns of dA (fork_inputs) and [dGz|dGr]
          if (int rc = fork_copy(m, f, dWcat, dbcat, grads, st)) return rc;
          // recurrent weights: state_to_state = (h*r)^T dA ; state_to_gates = H_prev^T [dGz|dGr]
          float* gWs = grad(b + "/gatedrecurrent.state_to_state");
          float* gWg = grad(b + "/gatedrecurrent.state_to_gates");
          if (tc) {
            if (int rc = gemm_tn_tc(ws, hrT, dir * D, D, dPreT, cA, D, gWs, D, false, st)) return rc;
            if (int rc = gemm_tn_tc(ws, hpT[dir], 0, D, dPreT, cG, 2 * D, gWg, 2 * D, false, st)) return rc;
          } else {
            if (int rc = gemm_tn(ws, hr + dir * D, Dout, tp.pre + cA, N, rows, D, D, gWs, D, false, st)) return rc;
            if (int rc = gemm_tn(ws, hprev[dir], Dout, tp.pre + cG, N, rows, D, 2 * D, gWg, 2 * D, false, st)) return rc;
          }
          if (int rc = colsum(dh0 + (size_t)dir * B * D, B, D, D, grad(b + "/gatedrecurrent.initial_state"), false, st)) return rc;
        }
      }
      // gradient of the layer input = gradient of the (subsampled) output of the layer below, or of the bottom MLP's
      if (l > 0 || m->bottom.num_layers) {
        float* dX = ws.f32((size_t)rows * tp.Din);
        LVSR_CHECK(dX, "out of device memory (dX)");
        // dX = dPre . Wcat^T: the K-major form of the right-hand side [N = Din, K = 3 nd D] is Wcat itself
        if (int rc = input_grad(tp.pre, rows, N, m->Wcat[l].get(), tp.Din, dX, &plan[LVSR_ENC_DX])) return rc;
        dout = dX0 = dX;
      }
    }
    if (!m->bottom.num_layers) return 0;
    // the gradient of the bottom's output passes the multiplier that dropped it in the forward
    if (drop) if (int rc = dropout_apply(*drop, dX0, dX0, tape[0].T, B, tape[0].Din, st)) return rc;
    return bottom_backward(x, bottom_out, dX0, tape[0].T * B);
  }
};

// forward + backward of one batch on the parameters Param::dev points at and the weights packed from them
int forward_backward(lvsr_model* m, const float* x, const float* mask, const int64_t* labels, const float* lmask,
                     int32_t T, int32_t B, int32_t L, float gscale, float* cost_out, float* grads, void* stream,
                     const DropoutKey* drop, const Greedy* greedy) {
  if (int rc = check_ready(m)) return rc;
  LVSR_CHECK(x && labels && cost_out && grads && T > 0 && B > 0 && L > 0, "train_cost_and_grads: bad arguments");
  LVSR_CHECK(!lm_attached(m), "train_cost_and_grads: shallow fusion is inference only (detach the language model)");
  return TrainStep{m, static_cast<cudaStream_t>(stream), labels, lmask, grads, gscale, B, L, lvsr_encoded_length(m, T),
                   drop, m->reg.penalty_coof, greedy}
      .run(x, mask, T, cost_out);
}

// forward_backward on the parameter copy `copy` (flat layout): every parameter pointer is re-pointed at it and the
// kernel-side weights are re-packed from it; on every way out the pointers go back to the means and the handle is
// marked un-finalized, so any other entry point re-packs from the means first.
int forward_backward_on(lvsr_model* m, const float* copy, const float* x, const float* mask, const int64_t* labels,
                        const float* lmask, int32_t T, int32_t B, int32_t L, float gscale, float* cost_out, float* grads,
                        void* stream, const DropoutKey* drop, const Greedy* greedy) {
  struct Restore {
    lvsr_model* m;
    ~Restore() {
      for (Param& p : m->params) p.dev = m->flat.get() + p.offset;
      m->finalized = false;
      m->noise.stale = true;         // the step may still read the noisy packing on its own stream (check_ready)
    }
  } restore{m};
  for (Param& p : m->params) p.dev = const_cast<float*>(copy) + p.offset;
  if (int rc = finalize_on_stream(m, static_cast<cudaStream_t>(stream), false)) return rc;
  return forward_backward(m, x, mask, labels, lmask, T, B, L, gscale, cost_out, grads, stream, drop, greedy);
}

// lvsr_train_cost_and_grads, and with `greedy` its greedy-exploration form: the regularisation in force, then the step
// on the parameters it perturbs
int train_cost_and_grads(lvsr_model* m, const float* x, const float* mask, const int64_t* labels, const float* lmask,
                         int32_t T, int32_t B, int32_t L, float gscale, float* cost_out, float* grads, void* stream,
                         const Greedy* greedy) {
  LVSR_CHECK(!m || m->cfg.dec_stack == 1,
             "train_cost_and_grads: a stacked decoder (dec_stack %d) is inference only: no backward pass through the "
             "RecurrentStack", m ? m->cfg.dec_stack : 0);
  LVSR_CHECK(!m || !(tle_criterion(m) && lm_attached(m)),
             "train_cost_and_grads: shallow fusion is inference only: a task-loss handle with a language model decodes "
             "and scores (detach the language model)");
  if (int rc = bind_stream(m, static_cast<cudaStream_t>(stream))) return rc;
  const lvsr_model::Reg& r = m->reg;
  const bool weight_noise = r.level > 0.f;
  LVSR_CHECK(!(m->noise.on && (r.dropout || weight_noise || r.penalty_coof > 0.f)),
             "train_cost_and_grads: dropout, weight noise and the alignment penalty have no effect under adaptive noise "
             "(lvsr/main.py:425-437): turn them off (lvsr_train_set_regularization)");
  const DropoutKey key{r.seed, r.update, r.utt_offset};
  const DropoutKey* drop = r.dropout ? &key : nullptr;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (m->noise.on) {
    // adaptive weight noise (noise.cu): the step runs on p + eps sqrt(s2)
    if (int rc = noise_sample(m, st)) return rc;
    return forward_backward_on(m, m->noise.noisy, x, mask, labels, lmask, T, B, L, gscale, cost_out, grads, stream, drop,
                               greedy);
  }
  if (weight_noise) {
    // weight noise (noise.cu): the step runs on p + level eps, the attention's parameters as they are
    if (int rc = weight_noise_sample(m, st)) return rc;
    return forward_backward_on(m, r.noisy.get(), x, mask, labels, lmask, T, B, L, gscale, cost_out, grads, stream, drop,
                               greedy);
  }
  return forward_backward(m, x, mask, labels, lmask, T, B, L, gscale, cost_out, grads, stream, drop, greedy);
}

}  // namespace

extern "C" {

int lvsr_train_cost_and_grads(lvsr_model* m, const float* x, const float* mask, const int64_t* labels, const float* lmask,
                              int32_t T, int32_t B, int32_t L, float gscale, float* cost_out, float* grads, void* stream) {
  DeviceGuard device_guard(m);
  return train_cost_and_grads(m, x, mask, labels, lmask, T, B, L, gscale, cost_out, grads, stream, nullptr);
}

int lvsr_train_cost_and_grads_greedy(lvsr_model* m, const float* x, const float* mask, const int64_t* groundtruth,
                                     int32_t T, int32_t B, int32_t L, float gscale, float* cost_out, float* grads,
                                     int64_t* prediction, float* prediction_mask, void* stream) {
  DeviceGuard device_guard(m);
  LVSR_CHECK(m && groundtruth && prediction && prediction_mask && L > 0, "train_cost_and_grads_greedy: bad arguments");
  LVSR_CHECK(tle_criterion(m), "train_cost_and_grads_greedy: greedy exploration trains a task-loss criterion "
             "(mse_gain / mse_reward; lvsr_model_set_criterion)");
  LVSR_CHECK(m->reg.penalty_coof <= 0.f, "train_cost_and_grads_greedy: the alignment penalty pairs the L + %d generated "
             "steps with the L-row label mask (lvsr/main.py:411-417): it is undefined under greedy exploration",
             LVSR_GREEDY_EXTRA_STEPS);
  LVSR_CHECK(!m->reg.dropout, "train_cost_and_grads_greedy: dropout under greedy exploration picks one of two encoder "
             "applications in no defined order (lvsr/main.py:400-408)");
  const Greedy g{groundtruth, L, reinterpret_cast<long long*>(prediction), prediction_mask};
  return train_cost_and_grads(m, x, mask, prediction, prediction_mask, T, B, L + LVSR_GREEDY_EXTRA_STEPS, gscale,
                              cost_out, grads, stream, &g);
}

// Parameters with the WEIGHT role, the subjects of weight decay and max-norm (lvsr/main.py:418-420,493): Linear and
// LookupTable W and the recurrent matrices.  The conv filters carry no role of their own (lvsr/bricks/attention.py:31-33).
static bool is_weight_name(const std::string& name) {
  const std::string leaf = name.substr(name.rfind('.') + 1);
  return leaf == "W" || leaf == "state_to_state" || leaf == "state_to_gates";
}

int lvsr_train_apply_updates(lvsr_model* m, float* grads, float gscale, const lvsr_train_config* tc, void* stream) {
  DeviceGuard device_guard(m);
  LVSR_CHECK(m && grads && tc, "train_apply_updates: null argument");
  LVSR_CHECK(!(tc->decay_rate < 0.f || tc->decay_rate > 1.f), "decay rate needs to be in [0, 1]");   // B/algorithms/__init__.py:481-482
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_stream(m, st)) return rc;
  const long long n = m->flat_count;
  const int np = (int)m->params.size();
  lvsr_model::Noise& z = m->noise;
  // adaptive noise takes the gradients of the cost without the decay term (lvsr/main.py:425-437)
  LVSR_CHECK(!(z.on && tc->decay > 0.f), "train_apply_updates: weight decay has no effect under adaptive noise: pass decay = 0");
  if (!m->opt_desc) {
    std::vector<ParamDesc> h(np);
    for (int i = 0; i < np; ++i) {
      h[i].offset = m->params[i].offset;
      h[i].rows = (int)m->params[i].shape[0];
      h[i].cols = (int)(m->params[i].ndim == 2 ? m->params[i].shape[1] : 1);
      h[i].is_weight = is_weight_name(m->params[i].name) ? 1 : 0;
    }
    DeviceBuffer<void> opt_desc;
    DeviceBuffer<float> opt_scratch;
    LVSR_CUDA_OK(opt_desc.alloc(sizeof(ParamDesc) * np));
    LVSR_CUDA_OK(cudaMemcpyAsync(opt_desc.get(), h.data(), sizeof(ParamDesc) * np, cudaMemcpyHostToDevice, st));
    LVSR_CUDA_OK(cudaStreamSynchronize(st));         // h goes away on return (once per handle)
    LVSR_CUDA_OK(opt_scratch.alloc(1032 * sizeof(float)));
    m->opt_desc = std::move(opt_desc);               // both tables, or neither
    m->opt_scratch = std::move(opt_scratch);
  }
  auto lazy = [&](DeviceBuffer<float>& p) -> int {
    if (p) return 0;
    LVSR_CUDA_OK(p.alloc((size_t)n * sizeof(float)));
    LVSR_CUDA_OK(cudaMemsetAsync(p.get(), 0, (size_t)n * sizeof(float), st));
    return 0;
  };
  if (tc->use_momentum) if (int rc = lazy(m->opt_velocity)) return rc;
  if (tc->use_adadelta) { if (int rc = lazy(m->opt_ms_step)) return rc; if (int rc = lazy(m->opt_ms_dx)) return rc; }
  const ParamDesc* desc = static_cast<const ParamDesc*>(m->opt_desc.get());
  float* flat = m->flat.get();
  if (tc->decay > 0.f) {
    dim3 grid(64, np);
    add_decay_kernel<<<grid, 256, 0, st>>>(grads, flat, desc, np, 2.f * tc->decay / gscale);
    LVSR_LAUNCH_CHECK();
  }
  float* part = m->opt_scratch.get();
  float* norm = part + 1024;
  if (z.on) {
    // both gradient groups of adaptive noise (noise.cu), already multiplied by gscale; one clipping norm over both
    int nparts = 0;
    if (int rc = noise_gradients(m, grads, gscale, z.gls2, st, &nparts)) return rc;
    sqnorm_final_kernel<<<1, 32, 0, st>>>(z.norm_part, nparts, 1.f, norm, m->clip.get());
    LVSR_LAUNCH_CHECK();
    gscale = 1.f;
  } else {
    const int nparts = (int)std::min<long long>(1024, std::max<long long>(1, n / 4096));
    sqnorm_partial_kernel<<<nparts, 256, 0, st>>>(grads, n, part);
    LVSR_LAUNCH_CHECK();
    sqnorm_final_kernel<<<1, 32, 0, st>>>(part, nparts, gscale, norm, m->clip.get());
    LVSR_LAUNCH_CHECK();
  }
  StepArgs a = {};
  a.grads = grads; a.params = flat; a.velocity = m->opt_velocity.get(); a.ms_step = m->opt_ms_step.get();
  a.ms_dx = m->opt_ms_dx.get();
  a.norm = norm; a.n = n; a.gscale = gscale; a.decay = tc->decay; a.threshold = tc->gradient_threshold;
  a.clip = m->clip.get();
  a.use_momentum = tc->use_momentum; a.learning_rate = tc->scale; a.momentum = tc->momentum;
  a.use_adadelta = tc->use_adadelta; a.decay_rate = tc->decay_rate; a.epsilon = tc->epsilon;
  step_rules_kernel<<<grid1d(n, 256, 1184), 256, 0, st>>>(a);
  LVSR_LAUNCH_CHECK();
  if (z.on) {          // the same rules over the ls2 block, with its own optimizer state
    StepArgs b = a;
    b.grads = z.gls2; b.params = z.ls2; b.velocity = z.velocity; b.ms_step = z.ms_step; b.ms_dx = z.ms_dx;
    step_rules_kernel<<<grid1d(n, 256, 1184), 256, 0, st>>>(b);
    LVSR_LAUNCH_CHECK();
  }
  if (tc->max_norm > 0.f) {
    dim3 grid(32, np);
    max_norm_kernel<<<grid, 256, 0, st>>>(grads, flat, desc, tc->max_norm);
    LVSR_LAUNCH_CHECK();
  }
  float burn_mult = 1.f;
  if (tc->burn_in_steps > 0) {                         // lvsr/algorithms.py:35-43
    if (m->burn_in_left < 0) m->burn_in_left = tc->burn_in_steps;
    burn_mult = m->burn_in_left <= 0 ? 1.f : 0.f;
    m->burn_in_left = std::max<long long>(0, m->burn_in_left - 1);
  }
  m->reg.update++;     // the next step draws a fresh dropout mask and weight noise
  if (z.on) {          // RemoveNotFinite per tensor: every ls2 is a tensor of its own; no max-norm (PARAMETER role only)
    apply_update_pair_kernel<<<2 * np, 256, 0, st>>>(flat, grads, z.ls2, z.gls2, desc, np, burn_mult);
    LVSR_LAUNCH_CHECK();
    z.update++;
    z.sampled = false;
    // the next training forward packs the weights from its noisy copy; packing the means here as well would cost a
    // second re-pack per step, so they are packed when another entry point needs them (check_ready)
    z.stale = true;
    m->finalized = false;
    return 0;
  }
  apply_update_kernel<<<np, 256, 0, st>>>(flat, grads, desc, burn_mult);
  LVSR_LAUNCH_CHECK();
  if (m->reg.level > 0.f) {
    // as under adaptive noise: the next training forward packs its noisy copy, other entry points pack the means
    z.stale = true;
    m->finalized = false;
    return 0;
  }
  return finalize_on_stream(m, st, false);             // re-pack the kernel-side weights from the new parameters
}

int lvsr_train_gradient_norm(lvsr_model* m, float* norm_host) {
  LVSR_CHECK(m && norm_host && m->opt_scratch, "train_gradient_norm: no update has run yet");
  DeviceGuard device_guard(m);
  return copy_on_handle(m, norm_host, m->opt_scratch.get() + 1024, sizeof(float), cudaMemcpyDeviceToHost);   // after the update
}

int lvsr_train_reset(lvsr_model* m) {
  LVSR_CHECK(m, "null model");
  DeviceGuard device_guard(m);
  const size_t bytes = (size_t)m->flat_count * sizeof(float);
  cudaStream_t st = m->stream;     // after every update queued on the handle, before the next one
  if (m->opt_velocity) LVSR_CUDA_OK(cudaMemsetAsync(m->opt_velocity.get(), 0, bytes, st));
  if (m->opt_ms_step) LVSR_CUDA_OK(cudaMemsetAsync(m->opt_ms_step.get(), 0, bytes, st));
  if (m->opt_ms_dx) LVSR_CUDA_OK(cudaMemsetAsync(m->opt_ms_dx.get(), 0, bytes, st));
  if (m->noise.on) LVSR_CUDA_OK(cudaMemsetAsync(m->noise.velocity, 0, 3 * bytes, st));     // velocity | ms_step | ms_dx of ls2
  if (m->clip) LVSR_CUDA_OK(cudaMemcpyAsync(m->clip.get(), m->clip_init, sizeof(m->clip_init), cudaMemcpyHostToDevice, st));
  m->burn_in_left = -1;
  m->reg.update = 0;
  return 0;
}

int lvsr_train_set_adaptive_clipping(lvsr_model* m, const lvsr_adaptive_clipping* cfg) {
  LVSR_CHECK(m, "null model");
  DeviceGuard device_guard(m);
  static_assert(sizeof(m->clip_init) == CLIP_WORDS * sizeof(double), "clip_init holds the CLIP_* words");
  if (!cfg) {
    if (m->clip) {
      LVSR_CUDA_OK(cudaStreamSynchronize(m->stream));     // an update queued on the handle may still read the state
      m->clip.reset();
    }
    return 0;
  }
  LVSR_CHECK(cfg->initial_threshold > 0.0 && std::isfinite(cfg->initial_threshold),
             "adaptive clipping: initial_threshold must be > 0");
  LVSR_CHECK(cfg->decay_rate >= 0.0 && cfg->decay_rate <= 1.0, "adaptive clipping: decay_rate must be in [0, 1]");
  LVSR_CHECK(cfg->burnin_period > 0, "adaptive clipping: burnin_period must be > 0");
  double* c = m->clip_init;
  for (int i = 0; i < CLIP_WORDS; ++i) c[i] = 0.0;
  c[CLIP_THR] = c[CLIP_NEXT] = c[CLIP_THR0] = cfg->initial_threshold;
  c[CLIP_DECAY] = cfg->decay_rate;
  c[CLIP_BURNIN] = (double)cfg->burnin_period;
  if (!m->clip) LVSR_CUDA_OK(m->clip.alloc(sizeof(m->clip_init)));
  // after every update queued on the handle; the host image lives in the handle, so the copy needs no wait
  LVSR_CUDA_OK(cudaMemcpyAsync(m->clip.get(), c, sizeof(m->clip_init), cudaMemcpyHostToDevice, m->stream));
  return 0;
}

int lvsr_train_clipping_threshold(lvsr_model* m, double* threshold_host) {
  LVSR_CHECK(m && threshold_host, "null argument");
  LVSR_CHECK(m->clip, "adaptive clipping is off (lvsr_train_set_adaptive_clipping)");
  DeviceGuard device_guard(m);
  return copy_on_handle(m, threshold_host, m->clip.get() + CLIP_NEXT, sizeof(double), cudaMemcpyDeviceToHost);
}

}  // extern "C"
