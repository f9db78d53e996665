// Internal (C++) launch interfaces of the kernels behind the C ABI in include/lvsr_b200.h.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "lvsr_b200.h"

namespace lvsr {

// ---- gemm.cu ------------------------------------------------------------------------
struct GemmArgs {
  const float* A;          // row r lives at A + (r / rows_per_block) * block_stride + (r % rows_per_block) * lda
  int M, K;
  int rows_per_block;
  long long block_stride;
  int lda;
  const float* W;          // [K, N] row-major, leading dimension ldw
  int N, ldw;
  const float* bias;       // [N] or nullptr
  float* C;                // [M, N], leading dimension ldc
  int ldc;
  int accumulate;          // C += ... instead of C = ...
  int act;                 // LVSR_ACT_RELU / LVSR_ACT_TANH: C = act(...) after the bias and the accumulation; other: none
};
int gemm_bias(const GemmArgs& g, cudaStream_t stream);

inline GemmArgs make_gemm(const float* A, int M, int K, const float* W, int N, const float* bias,
                          float* C, bool accumulate = false) {
  GemmArgs g;
  g.A = A; g.M = M; g.K = K; g.rows_per_block = M > 0 ? M : 1; g.block_stride = 0; g.lda = K;
  g.W = W; g.N = N; g.ldw = N; g.bias = bias; g.C = C; g.ldc = N; g.accumulate = accumulate ? 1 : 0;
  g.act = LVSR_ACT_IDENTITY;
  return g;
}

// ---- gemm_tc.cu: wgmma / TMA path (3xTF32 split, or fp16 head/tail split when K % 64 == 0) -------------
bool gemm_tc_supported(int M, int N, int K);
int gemm_tc_kpad(int K);                 // contraction dimension as stored in the hi/lo operands (multiple of 32)
int split_weight_tf32(const float* W, int K, int N, float* Wt_hi, float* Wt_lo, cudaStream_t stream);
int transpose_split_tf32(const float* W, int K, int N, int ldw, float* hi, float* lo, cudaStream_t stream);
int split_tf32(const float* x, float* hi, float* lo, long long n, cudaStream_t stream);
int gemm_tc_presplit(const float* A_hi, const float* A_lo, int M, const float* B_hi, const float* B_lo, int N, int Kpad,
                     const float* bias, float* C, int ldc, int splits, long long split_stride, cudaStream_t stream);
int gemm_tc_splits_launched(int Kpad, int splits);   // how many partial outputs gemm_tc_presplit writes
int gemm_tc(const float* A, float* A_hi, float* A_lo, int M, int K, const float* Wt_hi, const float* Wt_lo, int N,
            const float* bias, float* C, int ldc, cudaStream_t stream);
bool gemm_f16_supported(int M, int N, int K);      // K a multiple of 64: fp16 operands, no padding
int split_weight_f16(const float* W, int K, int N, __half* Wt_head, __half* Wt_tail, int* ew, cudaStream_t stream);
int gemm_f16(const float* A, __half* A_head, __half* A_tail, int* ea, int M, int K, const __half* Wt_head,
             const __half* Wt_tail, const int* ew, int N, const float* bias, float* C, int ldc, cudaStream_t stream);
// The same product streamed behind the BiGRU scan that writes A (gemm_tc.cu: gemm_f16_stream_kernel): the kernel splits
// A itself, tile by tile, once the tile's rows are final.  A = the scan's output [ceil(T / k), B, K].  Two launches
// share one zeroed scheduling area `sync` (gemm_f16_stream_sync_ints(M) ints, zeroed before the scan starts): with
// `progress` set, right after the scan and beside it, on the SMs the scan leaves free; then with progress == null, on
// every SM, for the tiles the first launch did not claim.  Each adds the tiles it claimed to *tiles_done.
struct ProjStream {
  int* sync;
  const int* progress;     // gemm_f16_stream_progress(sync), handed to the scan (BiGruArgs::progress), or null
  int nscan, scan_cs;      // CTAs of the scan and CTAs per cluster (scan CTA i runs direction (i / scan_cs) % ndir)
  int ndir;                // directions of the scan (1: every CTA runs forward)
  int T, k, B;             // frames the scan runs, its subsampling, batch rows
  unsigned spin_limit;     // polls without progress before the launch beside the scan stops claiming
  int* tiles_done;
  int* claims;             // [3 x tiles] or null: the launch beside the scan records (m-tile + 1, forward and backward
                           // progress) of each tile it claims, at the progress it found the tile's rows final
};
bool gemm_f16_stream_supported(int M, int N, int K);
size_t gemm_f16_stream_sync_ints(int M);
int* gemm_f16_stream_progress(int* sync);
int gemm_f16_stream_max_scan_ctas();
int gemm_f16_stream(const float* A, __half* A_head, __half* A_tail, int* ea, int M, int K, const __half* Wt_head,
                    const __half* Wt_tail, const int* ew, int N, const float* bias, float* C, int ldc,
                    const ProjStream& ps, int grid, cudaStream_t stream);

// ---- bigru.cu -----------------------------------------------------------------------
struct BiGruArgs {
  const float* pre;        // [T*B, 3 ndir D]: per direction [inputs D | update-gate D | reset-gate D], fwd then bwd
  const float* mask;       // [T, B] view (time stride mask_tstride) or nullptr
  long long mask_tstride;
  const float *Wg_f, *Ws_f, *h0_f;   // forward  state_to_gates [D,2D], state_to_state [D,D], initial_state [D]
  const float *Wg_b, *Ws_b, *h0_b;   // backward (unused when ndir is 1)
  float* out;              // [ceil(T/subsample), B, ndir D] (forward units first)
  int T, B, D, subsample;
  int ndir;                // 2: both directions, 1: forward only (net.bidir False)
  // training only (both null for inference): the tape the backward scan reads
  float* tape;             // = pre, written in place: candidate c over the inputs slot, z / r over the gate slots
  float* hext;             // [(T+2), B, ndir D]: slot t+1 = states after time t; slot 0 (forward half) and slot T+1
                           // (backward half) = the broadcast initial states
  // optional, tensor-core kernel only: progress[cta] = time steps whose output stores that CTA has made visible at gpu
  // scope (published every few steps and after the last), for a projection streamed behind the scan
  int* progress;
};
bool bigru_supported(int D);
// what bigru_layer launched (lvsr_model_encoder_plan): kernel LVSR_ENC_BIGRU_*, rows and CTAs per cluster, clusters,
// the clusters of that kernel the device holds at once (occupancy query) and the waves that makes
struct BiGruPlan { int kernel, rb, cs, clusters, resident, waves; };
int bigru_plan(const BiGruArgs& a, BiGruPlan* plan);   // what bigru_layer would launch for a, without launching
int bigru_layer(const BiGruArgs& a, cudaStream_t stream, BiGruPlan* plan = nullptr);

// ---- bigru_bwd.cu: reverse-time scan of one layer (training) ------------------------------
struct BiGruBwdArgs {
  float* tape;             // [T*B, 3 ndir D] in: c | z | r per direction (forward's tape); out: dA | dGz | dGr
  const float* hext;       // [(T+2), B, ndir D] (see BiGruArgs)
  const float* mask;       // [T, B] view or nullptr
  long long mask_tstride;
  const float* dout;       // [ceil(T/subsample), B, ndir D] gradient of the layer's (subsampled) output
  const float *Wg_f, *Ws_f, *Wg_b, *Ws_b;
  float* hr_out;           // [T, B, ndir D]: h_prev * r (operand of the state_to_state gradient)
  float* dh0;              // [ndir, B, D]: gradient of the broadcast initial state, per direction and row
  int T, B, D, subsample;
  int ndir;                // as BiGruArgs::ndir
};
int bigru_layer_backward(const BiGruBwdArgs& a, cudaStream_t stream, int* cs_out = nullptr);   // *cs_out: CTAs per cluster

// ---- attention.cu -------------------------------------------------------------------
struct PriorParams {
  int type;                // LVSR_PRIOR_*
  double initial_begin, initial_end, min_speed, max_speed, before, after;
};

// Window of take_glimpses (lvsr/bricks/attention.py:123-163), computed on device.
//   win[0] = begin, win[1] = end (global cut); lohi[2r], lohi[2r+1] = per-row strict bounds
struct WindowArgs {
  const float* weights;    // [R, Tp] previous alignment
  const long long* step;   // [R] (only step[0] is used, by the expanding prior); may be nullptr (= 0)
  long long step_offset;   // added to step[0] (teacher forcing: the step index)
  int R, Tp;
  PriorParams prior;
  int* win;                // [2] (or [2 * nseg])
  float* lohi;             // [2R]
  // optional segmentation (batched beam search: one segment = the hypotheses of one utterance, which is the
  // reference's "batch" for the batch-global cut): rows [seg_start[s], seg_start[s+1]) -> win[2s], win[2s+1]
  const int* seg_start;    // [nseg + 1] or nullptr (one segment = all rows)
  int nseg;
  const int* seg_len;      // [nseg] valid encoded frames of the segment's utterance (<= Tp) or nullptr (= Tp)
};
int attention_window(const WindowArgs& a, cudaStream_t stream);

struct AttStepArgs {
  const float* P;          // [Tp, U, M] preprocessed attended
  const float* H;          // [Tp, U, E] attended
  const float* maskH;      // [Tp, U]
  const int* row_utt;      // [R] or nullptr (identity)
  const float* q;          // [R, M]  states . W_state
  const float* w_prev;     // [R, Tp]
  const int* win;          // [2] from attention_window ([2 * nseg] with row_seg)
  const int* row_seg;      // [R] segment of each row or nullptr (all rows share win[0..1])
  const float* lohi;       // [2R]
  const float* filt;       // [K, 2n+1]
  const float* Wh;         // [K, M]
  const float* v;          // [M]
  float v_bias;            // energy bias (only when normalizer != softmax)
  float* w_out;            // [R, Tp]
  float* e_out;            // [R, Tp]
  float* ctx;              // [R, E]
  int R, U, Tp, M, E, K, n, normalizer;
};
// location = false: content-only attention (no previous alignment, conv or handler; filt / Wh / K / n unused, e_out
// receives zeros).  *cs_out = the cluster size launched.
int attention_step(const AttStepArgs& a, bool location, int* cs_out, cudaStream_t stream);
int attention_max_cluster();

// ---- decoder.cu ---------------------------------------------------------------------
// out[R,N] = epilogue( sum over the operands, in order, of X[R,K].W[K,ncols] (columns < ncols only) + add[arow[r]] )
enum { DENSE_PLAIN = 0, DENSE_GATES = 1, DENSE_CAND = 2, DENSE_ACT = 3 };
struct DenseOperand {
  const float* X; int K, ldx;   // X [R, K], row stride ldx; null: no operand
  const float* W; int ncols;    // W [K, ncols], ncols <= N
};
struct DenseArgs {
  DenseOperand op[3];
  const float* add;        // [*, N] addend rows or nullptr
  const long long* arow;   // [R] row index into add (labels) or nullptr (identity)
  long long add_rows;      // rows of `add` when arow is given (0 = unknown): indices are clamped into the table
  int R, N, mode;
  // DENSE_PLAIN: out[R,N]; DENSE_ACT: out[R,N] = act(acc + bias) (a readout hidden layer, act LVSR_ACT_*)
  float* out;
  const float* bias; int act;
  // DENSE_GATES (N = 3C): cols [0,C) update -> z[R,C]; [C,2C) reset -> hr[R,C] = s*r; [2C,3C) -> ai[R,C]
  // DENSE_CAND  (N = C):  c = tanh(acc + ai); s' = c*z + s*(1-z); optional row mask blend -> out[R,C], row stride ld_out
  const float* s; int ld_s;   // [R, C] current states, row stride ld_s
  float* z; float* hr; float* ai;
  const float* rmask;      // [R] or nullptr
  int C, ld_out;
};
int dense_step(const DenseArgs& a, cudaStream_t stream);

// readouts -> -log softmax.  merged [R, Cpm] (already merge + nothing else): adds bias, maxout/relu,
// Linear(Cpm/pieces -> V), log-softmax; writes either all V costs or the cost of labels[r].
struct ReadoutArgs {
  const float* merged;     // [R, Cpm]
  const float* b_pm;       // [Cpm]
  const float* Wo;         // [Cpm/pieces, V]
  const float* bo;         // [V]
  int R, Cpm, pieces, V, act;   // act: LVSR_ACT_*
  const long long* labels; // [R] or nullptr
  const float* lmask;      // [R] or nullptr (multiplies the picked cost)
  float* costs_all;        // [R, V] or nullptr
  float* costs_picked;     // [R] or nullptr
  const unsigned* poison;  // optional launch-status word of the producer: non-zero -> every cost is NaN
  // shallow fusion (ShallowFusionReadout + LMEmitter, lvsr/bricks/language_models.py): with lm_add the cost is -x,
  // x = am_beta * logits (log-softmaxed if norm_am) + lm_weight * (-lm_add, log-softmaxed if norm_lm), log-softmaxed
  // again if norm_tot.  lm_add == nullptr: the plain SoftmaxEmitter cost.
  const float* lm_add;     // [R, V] or nullptr
  float lm_weight, am_beta;
  int norm_am, norm_lm, norm_tot;
  // RewardRegressionEmitter (lvsr/bricks/__init__.py:119-202): the costs are -readouts, no log-softmax; with lm_add the
  // readouts are the fused x above, so the costs are -x as under the SoftmaxEmitter
  int tle;
};
int readout_costs(const ReadoutArgs& a, cudaStream_t stream);
// Shared memory the readout kernels stage per CTA of 8 rows for a last hidden width H: readout_kernel (decoder.cu) and
// the training step's readout_bwd_kernel (train_kernels.cuh), each at most READOUT_SMEM_LIMIT
constexpr size_t READOUT_SMEM_LIMIT = 48 * 1024;
constexpr size_t readout_smem_bytes(int H) { return (size_t)8 * H * sizeof(float); }
constexpr size_t readout_bwd_smem_bytes(int H) { return (size_t)8 * (H + 128) * sizeof(float); }

// ---- tle.cu: task loss estimation, RewardOp + RewardRegressionEmitter.cost (lvsr/ops.py:236-294,
// lvsr/error_rate.py:11-112, lvsr/bricks/__init__.py:135-184) --------------------------------------------------------
// rewards / gains [L, B, V] of prediction [L, B] against groundtruth [Lg, B] (int64, symbols in [0, V)), one CTA per
// utterance.  dist: tle_dist_ints(Lg, L, B) ints of scratch.  status: the lowest utterance whose groundtruth holds no
// eos is atomicMin-ed into it (the caller sets it to LVSR_TLE_OK first); that utterance's rows are not written.
enum : unsigned { LVSR_TLE_OK = 0xffffffffu };
enum { LVSR_TLE_GAIN = 1, LVSR_TLE_REWARD = 2 };   // the mse_gain / mse_reward losses (LVSR_CRITERION_MSE_*)
size_t tle_dist_ints(int Lg, int L, int B);
int tle_matrices(const long long* groundtruth, int Lg, const long long* prediction, int L, int B, int V, int eos,
                 int* dist, float* rewards, float* gains, unsigned* status, cudaStream_t stream);
// costs [L, B] of the loss `criterion` (LVSR_TLE_*) from the emitter costs neg_readouts [L*B, V] (= -readouts), the
// matrices above and prediction [L, B]; multiplied by lmask [L, B] when it is given.  One warp per utterance.
int tle_loss(int criterion, const float* neg_readouts, const float* rewards, const float* gains,
             const long long* prediction, const float* lmask, int L, int B, int V, float min_reward, float* costs,
             cudaStream_t stream);
// dlogits [L*B, V] = gscale * d sum(tle_loss costs) / d readouts, from the same inputs; row_sum: L*B doubles of scratch
int tle_loss_grad(int criterion, const float* neg_readouts, const float* rewards, const float* gains,
                  const long long* prediction, const float* lmask, int L, int B, int V, float min_reward, float gscale,
                  double* row_sum, float* dlogits, cudaStream_t stream);
// One greedy step from the emitter costs neg_readouts [B, V]: out [B] = the arg-max of the readouts, out_mask [B] =
// alive [B] (1 until eos has been emitted), then alive is cleared where out is eos
int tle_greedy_pick(const float* neg_readouts, int B, int V, int eos, float* alive, long long* out, float* out_mask,
                    cudaStream_t stream);

// ---- lm.cu: FST language model states (float64 weights, at most LVSR_LM_MAX_STATES per hypothesis) --------------
enum { LVSR_LM_TOO_MANY_STATES = 1, LVSR_LM_CLOSURE_CAP = 2, LVSR_LM_CYCLE = 3 };   // status word codes
struct LmFst {
  const long long* off;    // [num_states + 1] arc offsets
  const int* label;        // [num_arcs] NN label + 1, 0 = epsilon; sorted by (label, next) within a state
  const int* next;         // [num_arcs]
  const float* weight;     // [num_arcs]
  int start, V;
  float no_transition_cost;
  unsigned* status;        // first error of a launch (LVSR_LM_*), zeroed by the caller
};
// One warp per row: the set of row parent[r] (identity if null) advanced by symbols[r], or, with symbols == nullptr,
// expand({start}); writes the set (padded with -1 / 0) and its cost row add_out [R, V].
int lm_step(const LmFst& f, int R, const int* src_states, const double* src_weights, const int* parent,
            const long long* symbols, int* states_out, double* weights_out, float* add_out, cudaStream_t stream);
// Teacher forcing: add [L, B, V], row (i, b) = the cost row in force before labels[i, b]; masked labels are skipped.
int lm_path(const LmFst& f, int L, int B, const long long* labels, const float* lmask, float* add, cudaStream_t stream);
// dst row r = src row idx[r] of the (states, weights, add) triple
int lm_gather(int* states, double* weights, float* add, const int* src_states, const double* src_weights,
              const float* src_add, const int* idx, int Rn, int V, cudaStream_t stream);

// ---- dec_scan.cu: persistent teacher-forced decoder -----------------------------------
// The caller's inputs.  The hand-over protocol between the kernel's CTAs is dec_scan.cu's alone: run_dec_scan takes
// the per-step hand-over buffers from the workspace and pre-fills them, s_all and ctx_all with the sentinel.
struct DecScanInputs {
  const float *P, *H, *maskH;          // [Tp,B,M], [Tp,B,E], [Tp,B]
  const float *filt, *Wh, *v;          // attention constants
  float v_bias;
  PriorParams prior;
  const float* Wb1;                    // [E+C, 3C]: rows <E = distribute [gates|inputs], rows >=E = [state_to_gates | 0]
  const float* Wstate;                 // [C, C]
  const float* Ws;                     // [C, M]
  const float* FF;                     // [(V+1), 3C] fork(feedback(y)), gate columns first
  const long long* labels;             // [L, B]
  const float* lmask;                  // [L, B] or nullptr
  float* s_all;                        // [(L+1), B, C]; s_all[0] = initial states on entry
  float* ctx_all;                      // [L, B, E]
  const float* w0;                     // [B, Tp] initial alignment
  float* w_all;                        // [L, B, Tp] alignments: the caller's weights output, or nullptr (scratch)
  float* e_seq;                        // [L, B, Tp] or nullptr
  float* e_scratch;                    // [B, Tp]
  unsigned* status;                    // launch status word (common.cuh: LVSR_FLOW_*), zeroed by the caller
  int Tp, B, L, M, E, C, K, n, normalizer;
  int V;                               // num_phonemes: the feedback table FF has V + 1 rows
};
struct Arena;
// Runs the persistent decoder when a plan fits (*ran = true, plan[LVSR_PLAN_*] describe it); else *ran = false, only
// plan[LVSR_PLAN_MAX_CLUSTERS] is set and the caller runs the step-wise kernels.  location = false: content attention.
int run_dec_scan(const DecScanInputs& in, bool location, Arena& ws, int32_t* plan, bool* ran, cudaStream_t stream);

// small utility kernels
int fill_f32(float* p, long long n, float v, cudaStream_t stream);
int fill_i64(long long* p, long long n, long long v, cudaStream_t stream);
int broadcast_rows(float* dst, const float* src, int R, int N, cudaStream_t stream);   // dst[r,:] = src[:]
int onehot_rows(float* dst, int R, int N, cudaStream_t stream);                         // dst[r,:] = e_0
int gather_rows(float* dst, const float* src, const int* idx, int Rn, int N, cudaStream_t stream);   // dst[r,:] = src[idx[r],:]
int gather_i64(long long* dst, const long long* src, const int* idx, int Rn, long long inc, cudaStream_t stream);
// k smallest of cost_so_far[r] + neglogp[r, v] over the rows of each segment (B/search.py:341-344)
int segment_topk(const float* neglogp, const float* cost_so_far, const int* seg_start, int nseg, int V, int k,
                 int* top_parent, int* top_symbol, float* top_cost, int* top_count, cudaStream_t stream);
int add_bias_rows(float* dst, const float* src, const float* bias, int R, int N, cudaStream_t stream);   // dst[r,:] = src[r,:] + bias
int add_i64(long long* dst, const long long* src, int n, long long inc, cudaStream_t stream);
int gather_time_subsample(float* dst, const float* src, int Tout, int k, long long row_elems,
                          cudaStream_t stream);                                         // dst[t] = src[t*k]

}  // namespace lvsr
