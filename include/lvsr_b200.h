/*
 * lvsr_b200.h -- C ABI of the H100-native attention-lvcsr hot path.
 *
 * The reference (rizar/attention-lvcsr) has no FFI of its own on this path: Theano
 * generates and compiles C at run time and the "operator ABI" is the set of compiled
 * theano.function objects that Blocks/lvsr call.  Each entry point below replaces one
 * of those compiled functions 1:1 (SURVEY.md section 8b, tier b3); the reference-side
 * binding a maintainer would add is a ctypes stub, shown in INTEGRATION.md.
 *
 * Conventions
 *   - plain C: opaque handle, raw pointers, sizes.  No torch / C++ types.
 *   - all tensors are TIME-MAJOR and contiguous, float32 unless noted, exactly the
 *     layouts the reference feeds its compiled functions
 *     (lvsr/datasets/__init__.py:22-29,308; lvsr/bricks/recognizer.py:129-133,353-361).
 *   - `*_dev` pointers are device pointers on the model's GPU, `*_host` are host pointers.
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream); blocking and
 *     non-blocking streams are both fine.  A call that takes a stream is ordered on it.  The
 *     handle is bound to the stream of its last such call: a call on a different stream first
 *     synchronises the previous one, so the handle's workspace, device words and parameters are
 *     never used from two streams at once.  The caller orders its own buffers between streams,
 *     and keeps the bound stream alive until the handle's next call on another one.
 *   - host calls without a stream (get/set_param, finalize, status, train_gradient_norm,
 *     get/set_noise_param) act after all work queued on the handle: they synchronise its bound
 *     stream.  train_reset is enqueued on that stream without waiting.
 *   - calls with a stream do not synchronise, except: the `*_host` convenience calls (copy H2D,
 *     compute, copy D2H, synchronise the stream); a call that needs a larger workspace than the
 *     handle holds (it is regrown); the first call after parameters changed (it re-packs the
 *     weights, like lvsr_model_finalize); the LM calls noted below; and, with the logistic or
 *     relu normaliser, the call that re-packs the weights after an update, which reads the energy
 *     bias back to the host as a kernel argument: lvsr_train_apply_updates without adaptive
 *     noise, lvsr_train_cost_and_grads (for the noisy bias) with it.
 *   - every call returns 0 on success, non-zero on error; lvsr_last_error() then
 *     describes the failure (thread-local).
 *   - one model handle per GPU; a handle is not thread-safe.
 */
#ifndef LVSR_B200_H
#define LVSR_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct lvsr_model lvsr_model;

enum { LVSR_MAX_LAYERS = 8 };
enum { LVSR_NORM_SOFTMAX = 0, LVSR_NORM_LOGISTIC = 1, LVSR_NORM_RELU = 2 };
enum { LVSR_ACT_MAXOUT = 0, LVSR_ACT_RELU = 1, LVSR_ACT_TANH = 2, LVSR_ACT_IDENTITY = 3 };
enum { LVSR_PRIOR_EXPANDING = 0, LVSR_PRIOR_WINDOW_MEAN = 1, LVSR_PRIOR_WINDOW_MEDIAN = 2 };
/* attention_type (lvsr/bricks/recognizer.py:261-277): SequenceContentAndConvAttention ("conv_att") or
 * SequenceContentAttention ("cont_att", libs/blocks/blocks/bricks/attention.py:259-414).  Content attention has no
 * conv, handler, window or energy bias: conv_n, conv_num_filters, energy_normalizer and the prior are ignored, as the
 * reference does not pass them to that brick; every encoded frame of an utterance is attended. */
enum { LVSR_ATT_CONTENT_AND_CONV = 0, LVSR_ATT_CONTENT = 1 };

/* The subset of config['net'] the path depends on
 * (SpeechRecognizer.__init__, lvsr/bricks/recognizer.py:176-204). */
typedef struct {
  int32_t num_features;            /* F: input_dims['recordings']                     */
  int32_t num_layers;              /* len(dims_bidir)                                  */
  int32_t dims_bidir[LVSR_MAX_LAYERS];
  int32_t subsample[LVSR_MAX_LAYERS];
  int32_t dim_dec;                 /* C                                                */
  int32_t dim_matcher;             /* M (defaults to dim_dec, recognizer.py:225-226)   */
  int32_t conv_n;                  /* n, filter length 2n+1                            */
  int32_t conv_num_filters;        /* K                                                */
  int32_t num_phonemes;            /* V; the lookup table has V+1 rows                 */
  int32_t dim_feedback;            /* Cfb (dim_dec unless dim_output_embedding)        */
  int32_t post_merge_dim;          /* post_merge_dims[0]                               */
  int32_t maxout_pieces;           /* num_pieces of Maxout, 1 otherwise                */
  int32_t post_merge_activation;   /* LVSR_ACT_* (reference default: Tanh)             */
  int32_t use_states_for_readout;
  int32_t energy_normalizer;       /* LVSR_NORM_*                                      */
  int32_t prior_type;              /* LVSR_PRIOR_*                                     */
  double prior_initial_begin, prior_initial_end, prior_min_speed, prior_max_speed;
  double prior_before, prior_after;
  int32_t one_of_n_feedback;       /* 0: LookupFeedback(V+1, dim_feedback) (embed_outputs=True, the default);
                                      1: OneOfNFeedback(V+1) (embed_outputs=False, lvsr/bricks/__init__.py:86-109;
                                      exp/wsj/configs/wsj_jan_new.yaml:46): feedback = one-hot, dim_feedback = V+1  */
  int32_t attention_type;          /* LVSR_ATT_* (0, the zeroed default: content_and_conv)                      */
  int32_t dec_stack;               /* GRU layers of the decoder: 1 (0, the zeroed default, reads as 1) or 2, a
                                      RecurrentStack with skip connections (lvsr/bricks/recognizer.py:250-259).  With 2
                                      the decoder state of a row is [s0 | s1], 2 * dim_dec floats, wherever the ABI
                                      takes or returns states; training refuses it (inference only).              */
} lvsr_config;

/* The bottom MLP of config['net']['bottom'] (SpeechBottom, lvsr/bricks/recognizer.py:105-157): with num_layers = k > 0
 * every frame passes x_{i+1} = act(x_i W_i + b_i), i = 0 .. k-1, before encoder layer 0, which then takes dims[k-1]
 * features.  x_0 is the recordings (num_features); activation is LVSR_ACT_RELU (Rectifier) or LVSR_ACT_TANH.  Its
 * parameters are "/recognizer/bottom/bottom/linear_<i>.W" [d_in, dims[i]] and ".b" [dims[i]], after the encoder's and
 * before the generator's in the parameter table.  num_layers = 0 is the Identity bottom (dims: []). */
enum { LVSR_MAX_BOTTOM = 4, LVSR_MAX_BOTTOM_DIM = 4096 };
typedef struct {
  int32_t num_layers;              /* k = len(dims), 0 .. LVSR_MAX_BOTTOM                                        */
  int32_t dims[LVSR_MAX_BOTTOM];   /* 1 .. LVSR_MAX_BOTTOM_DIM each                                              */
  int32_t activation;              /* LVSR_ACT_RELU or LVSR_ACT_TANH (the reference's default for None)          */
} lvsr_bottom_config;

const char* lvsr_last_error(void);
int lvsr_version(void);

/* ---- model life cycle ----------------------------------------------------------- */
/* SpeechRecognizer(**config['net']) + allocate(): lvsr/main.py:213-221. Uses the
 * CUDA device current on the calling thread. */
int lvsr_model_create(const lvsr_config* cfg, lvsr_model** out);
/* The same with a bottom MLP (NULL: none, which is lvsr_model_create).  Every entry point that takes recordings runs
 * it; a depth, width or activation outside lvsr_bottom_config's ranges is refused here. */
int lvsr_model_create_bottom(const lvsr_config* cfg, const lvsr_bottom_config* bottom, lvsr_model** out);
/* The same with the encoder's direction count (net.bidir, lvsr/bricks/__init__.py:54-78): bidir 1 is the bidirectional
 * encoder the two calls above build; bidir 0 makes every layer l one forward-only GatedRecurrent
 * ("/recognizer/encoder/with_fork<l>/..."), layer l + 1 takes dims_bidir[l] features and the encoded width is
 * dims_bidir[num_layers - 1].  Any other value is refused before any device work.  Added within version 104: detect it
 * by its symbol. */
int lvsr_model_create_encoder(const lvsr_config* cfg, const lvsr_bottom_config* bottom, int32_t bidir, lvsr_model** out);

/* The readout's post-merge MLP of config['net']['post_merge_dims'] = [d_1 .. d_k] (lvsr/bricks/recognizer.py:305-320):
 * Bias(d_1) -> act -> MLP([act] * (k-1) + [Identity], [d_1 .. d_k, V]), act = cfg->post_merge_activation.  With
 * h_0 = act(merged + post_merge/bias.b), h_j = act(h_{j-1} W_{j-1} + b_{j-1}) for j = 1 .. k-1 and the logits
 * h_{k-1} W_{k-1} + b_{k-1}; W_j = "/recognizer/generator/readout/post_merge/mlp/linear_<j>.W" [d_{j+1}, d_{j+2}] (the
 * last [d_k, V]), each Linear's .b before its .W in the parameter table, as Blocks initialises them.  num_layers = k:
 * 1 .. LVSR_MAX_READOUT; dims[0] must equal cfg->post_merge_dim.  Above depth 1 every width is a multiple of 8, the
 * activation is not Maxout with more than one piece (the reference's MLP takes d_j / pieces inputs and its Maxout
 * divides them again), and d_k is at most lvsr_readout_max_width(). */
enum { LVSR_MAX_READOUT = 4 };
typedef struct {
  int32_t num_layers;              /* k = len(post_merge_dims), 1 .. LVSR_MAX_READOUT                            */
  int32_t dims[LVSR_MAX_READOUT];  /* d_1 .. d_k                                                                 */
} lvsr_readout_config;
/* The widest last hidden layer the readout kernels (forward and training backward) stage in shared memory. */
int lvsr_readout_max_width(void);
/* lvsr_model_create_encoder with the readout's post-merge depth: readout NULL (or num_layers 1) is depth 1, which is
 * lvsr_model_create_encoder itself.  A readout outside the rules above is refused before any device work.  Added within
 * version 104: detect it by its symbol. */
int lvsr_model_create_readout(const lvsr_config* cfg, const lvsr_bottom_config* bottom, int32_t bidir,
                              const lvsr_readout_config* readout, lvsr_model** out);
int lvsr_model_destroy(lvsr_model* m);

/* Parameter table in Blocks order/names ("/recognizer/encoder/bidir0/forward/fork/fork_inputs.W"
 * ...): Selector.get_parameters, libs/blocks/blocks/select.py:160-220. */
int lvsr_model_num_params(const lvsr_model* m);
const char* lvsr_model_param_name(const lvsr_model* m, int index);
int lvsr_model_param_shape(const lvsr_model* m, int index, int64_t shape[2], int32_t* ndim);
/* Model.set_parameter_values / get_parameter_values (lvsr/bricks/recognizer.py:408-412). */
int lvsr_model_set_param(lvsr_model* m, const char* name, const float* values_host, int64_t count);
int lvsr_model_get_param(const lvsr_model* m, const char* name, float* values_host, int64_t count);
/* All parameters live in ONE device allocation ("flat" layout: parameter i at float offset
 * lvsr_model_param_offset, 256-byte aligned, padding zero).  Gradients, optimizer state and the
 * gradient all-reduce of the training step use buffers of the same layout and size. */
int64_t lvsr_model_flat_size(const lvsr_model* m);
int lvsr_model_param_offset(const lvsr_model* m, int index, int64_t* offset, int64_t* count);
float* lvsr_model_flat_params(lvsr_model* m);     /* device pointer; call lvsr_model_finalize after writing through it */
/* Re-derive the packed kernel-side weights after parameters changed. */
int lvsr_model_finalize(lvsr_model* m);
/* Launch status of the persistent teacher-forced decoder of the LAST lvsr_cost_matrix call on this
 * handle (synchronises the handle's stream): 0 = ok, 2 = a hand-over value never arrived within the
 * polling limit, 3 = the launch lost its cluster shape.  On a non-zero status the costs of that call
 * are NaN (never plausible garbage); lvsr_recognizer_cost_host re-runs such a call on the step-wise
 * kernels by itself and counts it in *stepwise_fallbacks (may be NULL).  No reference counterpart:
 * Theano raises from inside the compiled function instead. */
int lvsr_model_status(lvsr_model* m, int32_t* launch_status, int64_t* stepwise_fallbacks);
/* Plan of the decoder (host state, no synchronisation): out[LVSR_PLAN_*] describes the LAST lvsr_cost_matrix on this
 * handle (training forwards included), all zero except MAX_CLUSTERS when it ran on the step-wise kernels, and
 * out[LVSR_PLAN_ATT_CS] the cluster size of the last attention step (state functions, beam search and the step-wise
 * fallback; 0 before the first).  The plan-forcing switches LVSR_DEC_CS, LVSR_DEC_LAYOUT, LVSR_DEC_HANDLER and
 * LVSR_ATT_CS (DESIGN §7) narrow what the planners may choose; this report says what they did choose. */
enum {
  LVSR_PLAN_RAN = 0,          /* 1: the persistent decoder ran                                                 */
  LVSR_PLAN_KERNEL = 1,       /* LVSR_PLAN_DEC_*                                                               */
  LVSR_PLAN_CS = 2,           /* CTAs per row cluster                                                          */
  LVSR_PLAN_GRID = 3,         /* CTAs launched                                                                 */
  LVSR_PLAN_NISL = 4,         /* islands (0: global layout)                                                    */
  LVSR_PLAN_NRG = 5,          /* 16-row groups of the global layout (1 in islands)                             */
  LVSR_PLAN_NCG = 6,          /* column groups of the dense tiles                                              */
  LVSR_PLAN_NC1 = 7,          /* columns per CTA: gate tile, candidate tile, query tile                        */
  LVSR_PLAN_NC2 = 8,
  LVSR_PLAN_NC3 = 9,
  LVSR_PLAN_TC_CAP = 10,      /* positions per rank (ceil(T'/cs))                                              */
  LVSR_PLAN_WH_ROWS = 11,     /* handler rows in shared memory: 16 (padded) or K (compact)                     */
  LVSR_PLAN_RED_ALIAS = 12,   /* 1: the dense tiles' scratch shares the attention reduction scratch            */
  LVSR_PLAN_ATT_CS = 13,      /* cluster size of the last attention step launch                                */
  LVSR_PLAN_MAX_CLUSTERS = 14,/* answer of the planner's last occupancy query (0: none made)                   */
  LVSR_PLAN_L2_KB = 15        /* KB of P and H per step the decoder loads with L2 evict-first (0: plain loads)  */
};
enum { LVSR_PLAN_STEPWISE = 0, LVSR_PLAN_DEC_SCAN = 1, LVSR_PLAN_DEC_SCAN_COMPACT = 2, LVSR_PLAN_DEC_CONTENT = 3 };
int lvsr_model_decoder_plan(const lvsr_model* m, int32_t out[16]);
/* Plan of the encoder (host state, no synchronisation), per layer 0 <= layer < num_layers: slots LVSR_ENC_PROJ ..
 * LVSR_ENC_T describe the LAST encoder forward on this handle (lvsr_encoder_forward, lvsr_recognizer_cost_host or the
 * forward of a training step), slots LVSR_ENC_BWD_CS .. LVSR_ENC_DX the backward pass of the LAST
 * lvsr_train_cost_and_grads (all zero before the first).  layer = -1 reports the last lvsr_preprocess (it also runs
 * inside every cost and training call) in LVSR_ENC_PROJ, LVSR_ENC_KPAD and LVSR_ENC_OPERANDS, every other slot zero.  The switches
 * LVSR_BIGRU_MMA, LVSR_BIGRU_RB and LVSR_NO_TC_GEMM (DESIGN §7; the last one is read by lvsr_model_finalize) force
 * the choices; this report says what ran. */
enum {
  LVSR_ENC_PROJ = 0,          /* fork projection GEMM: LVSR_ENC_PATH_*                                         */
  LVSR_ENC_KPAD = 1,          /* its contraction as the tensor-core GEMM stores it (0 on FFMA): unpadded on fp16
                                 operands (a multiple of 64), padded to a multiple of 32 on tf32 operands       */
  LVSR_ENC_BIGRU = 2,         /* LVSR_ENC_BIGRU_*: the scan kernel                                             */
  LVSR_ENC_TAPE = 3,          /* 1: the scan kept the tape of a training step                                  */
  LVSR_ENC_RB = 4,            /* batch rows per cluster                                                        */
  LVSR_ENC_CS = 5,            /* CTAs per cluster                                                              */
  LVSR_ENC_CLUSTERS = 6,      /* clusters launched (both directions)                                           */
  LVSR_ENC_RESIDENT = 7,      /* clusters of that kernel the device holds at once (occupancy query)            */
  LVSR_ENC_WAVES = 8,         /* ceil(clusters / resident)                                                     */
  LVSR_ENC_T = 9,             /* frames the layer scanned                                                      */
  LVSR_ENC_BWD_CS = 10,       /* CTAs per cluster of the reverse-time scan                                     */
  LVSR_ENC_WGRAD = 11,        /* weight gradients X^T dY: LVSR_ENC_PATH_*                                      */
  LVSR_ENC_WGRAD_SPLITS = 12, /* partial products the contraction over T_l * B rows was split into             */
  LVSR_ENC_WGRAD_KPAD = 13,   /* that contraction as the tensor-core operands store it (0 on FFMA)             */
  LVSR_ENC_DX = 14,           /* input gradient dY W^T: LVSR_ENC_PATH_* (NONE for layer 0 without a bottom MLP)*/
  LVSR_ENC_OPERANDS = 15      /* operands of the tensor-core projection GEMM: LVSR_ENC_OPS_*                   */
};
enum { LVSR_ENC_PATH_NONE = 0, LVSR_ENC_PATH_TC = 1, LVSR_ENC_PATH_FFMA = 2 };
/* LVSR_ENC_OPS_TF32X3: tf32 hi/lo split, three products; LVSR_ENC_OPS_F16X3: fp16 head/tail split of rows and columns
 * scaled by powers of two, three products (forward projections whose contraction is a multiple of 64) */
enum { LVSR_ENC_OPS_NONE = 0, LVSR_ENC_OPS_TF32X3 = 1, LVSR_ENC_OPS_F16X3 = 2 };
enum { LVSR_ENC_BIGRU_NONE = 0, LVSR_ENC_BIGRU_FFMA = 1, LVSR_ENC_BIGRU_MMA = 2 };
int lvsr_model_encoder_plan(const lvsr_model* m, int32_t layer, int32_t out[16]);
/* Projection of encoder layer 1 <= layer < num_layers in the LAST encoder forward (synchronises with the device):
 * out[0] = 1 when it ran beside the BiGRU scan of layer - 1, streamed tile by tile as the scan's output became final
 * (DESIGN §4; LVSR_ENC_OVERLAP=0 turns that off), else 0; out[1] / out[2] = its 128 x 128 output tiles computed beside
 * the scan / by the launch on every SM after it (both 0 when out[0] is 0).  Layer 0 always reports zeros. */
int lvsr_model_encoder_overlap(lvsr_model* m, int32_t layer, int32_t out[3]);
/* For such a layer (out[0] == 1): per output tile c in claim order, out[3 c .. 3 c + 2] = (m-tile + 1, forward and backward
 * scan progress) at which the launch beside the scan found the tile's rows final and claimed it, zeros for the tiles
 * the launch after the scan did; count ints, at most 3 x the layer's tiles.  Synchronises with the device. */
int lvsr_model_encoder_overlap_claims(lvsr_model* m, int32_t layer, int32_t* out, int64_t count);

/* ---- encoder: BeamSearch.context_computer / Encoder.apply -------------------------
 * (libs/blocks/blocks/search.py:97-99; lvsr/bricks/__init__.py:71-78).
 * recordings [T,B,F], mask [T,B] (NULL = no mask) -> attended [T',B,E], attended_mask [T',B]
 * with T' = lvsr_encoded_length(T), E = 2*dims_bidir[last]. */
int lvsr_encoded_length(const lvsr_model* m, int32_t T);
int lvsr_encoded_dim(const lvsr_model* m);
int lvsr_encoder_forward(lvsr_model* m, const float* recordings_dev, const float* mask_dev,
                         int32_t T, int32_t B, float* attended_dev, float* attended_mask_dev,
                         void* stream);

/* attention.preprocess: lvsr/bricks/attention.py:228-230. attended [T',U,E] -> [T',U,M]. */
int lvsr_preprocess(lvsr_model* m, const float* attended_dev, int32_t Tp, int32_t U,
                    float* preprocessed_dev, void* stream);

/* ---- teacher-forced decoder: generator.cost_matrix --------------------------------
 * (libs/blocks/blocks/bricks/sequence_generators.py:254-326).
 * labels int64 [L,B], every entry in [0, num_phonemes) -- device memory, NOT range-checked here
 * (lvsr_recognizer_cost_host checks its host copy); labels_mask [L,B] or NULL.  Outputs: costs [L,B]; optional (NULL to
 * skip) weights [L,B,T'], energies [L,B,T'], states [L,B,S] (= s_{i-1}; S = dec_stack * C, [s0 | s1] rows with
 * dec_stack 2), weighted_averages [L,B,E].  dec_stack 2 always runs on the step-wise kernels. */
int lvsr_cost_matrix(lvsr_model* m, const float* attended_dev, const float* attended_mask_dev,
                     int32_t Tp, int32_t B, const int64_t* labels_dev, const float* labels_mask_dev,
                     int32_t L, float* costs_dev, float* weights_dev, float* energies_dev,
                     float* states_dev, float* weighted_averages_dev, void* stream);

/* ---- training criterion: log-likelihood or task loss estimation --------------------------------------------------
 * (lvsr/bricks/recognizer.py:285-297).  A handle starts with log_likelihood (SoftmaxEmitter, initial output
 * num_phonemes).  mse_gain / mse_reward switch it to RewardRegressionEmitter (lvsr/bricks/__init__.py:119-202):
 *   - every emitter cost (lvsr_logprobs, the beam search) is -readouts, without a log-softmax;
 *   - lvsr_cost_matrix returns the loss rows of RewardOp's matrices (lvsr/ops.py:236-294) times the label mask:
 *       mse_gain    sum_v (r - max(G, min_reward))^2
 *       mse_reward  sum_v (r + sum_{1<=s<=t} r[s, y_s] - R)^2
 *     with the labels as their own groundtruth (lvsr_cost_matrix_groundtruth takes another one);
 *   - lvsr_initial_states and the beam search start from initial_output (the reference's 0).
 * A groundtruth without eos_label makes the cost call fail naming the utterance; the call synchronises its stream to
 * find out.  lvsr_train_cost_and_grads trains it with imitative exploration (the labels are the prediction),
 * lvsr_train_cost_and_grads_greedy with greedy exploration.
 * With a language model attached (in either order with lvsr_model_set_lm) the readouts r become the fused readouts x
 * of shallow fusion (below): every emitter cost is -x, the same row the log-likelihood emitter writes under fusion,
 * and the losses above take x in place of r, with the LM rows along the labels (the prediction).  Both training entry
 * points refuse such a handle before any device work.
 * Callers that must run on an older library detect the entry point by its symbol. */
enum { LVSR_CRITERION_LOG_LIKELIHOOD = 0, LVSR_CRITERION_MSE_GAIN = 1, LVSR_CRITERION_MSE_REWARD = 2 };
typedef struct {
  int32_t name;                    /* LVSR_CRITERION_*                                           */
  int32_t eos_label;               /* the groundtruth's end symbol, in [0, num_phonemes)         */
  int32_t initial_output;          /* first output of generation and search, in [0, num_phonemes] */
  double min_reward;               /* mse_gain's floor of the gains (reference default -1.0)     */
} lvsr_criterion;
int lvsr_model_set_criterion(lvsr_model* m, const lvsr_criterion* criterion);
/* lvsr_cost_matrix with the prediction `labels` scored against groundtruth_dev [Lg, B] (int64; NULL: the labels) by
 * the task-loss criterion, as SpeechRecognizer.analyze does (lvsr/bricks/recognizer.py:423-494).  Under
 * log_likelihood the groundtruth is not read. */
int lvsr_cost_matrix_groundtruth(lvsr_model* m, const float* attended_dev, const float* attended_mask_dev,
                                 int32_t Tp, int32_t B, const int64_t* labels_dev, const float* labels_mask_dev,
                                 int32_t L, const int64_t* groundtruth_dev, int32_t Lg, float* costs_dev,
                                 float* weights_dev, float* energies_dev, float* states_dev,
                                 float* weighted_averages_dev, void* stream);
/* RewardOp alone: rewards_dev and gains_dev [L, B, num_phonemes] (float32, integer values) of prediction_dev [L, B]
 * against groundtruth_dev [Lg, B], with the eos_label of the handle's criterion.  Synchronises the stream. */
int lvsr_tle_matrices(lvsr_model* m, const int64_t* groundtruth_dev, int32_t Lg, const int64_t* prediction_dev,
                      int32_t L, int32_t B, float* rewards_dev, float* gains_dev, void* stream);

/* ---- alignment statistics of validation: weights_entropy and weights_penalty -------------------------------------
 * (lvsr/expressions.py:4-25 as lvsr/main.py:385-388 monitors them) of the weights lvsr_cost_matrix writes,
 * weights [L,B,T'], labels_mask [L,B] (NULL = all ones).  out_dev (float64, device):
 *   out[0] = sum_{i,b} mask[i,b] sum_t w log(w + 1e-7)
 *   out[1] = sum_{i>=1,b} mask[i,b] sum_t max(C_i[t] - C_{i-1}[t], 0),  C_i[t] = sum_{t'<=t} w[i,b,t']
 * One launch; float64 sums in a fixed order, so the result is deterministic.  T' is limited by the shared memory of a
 * CTA (8 bytes per position: about 29000 on an H100). */
int lvsr_alignment_stats(lvsr_model* m, const float* weights_dev, const float* labels_mask_dev, int32_t L, int32_t B,
                         int32_t Tp, double* out_dev, void* stream);

/* ---- the BeamSearch state functions (libs/blocks/blocks/search.py:101-142) ---------
 * R rows (beam hypotheses); row r attends utterance row_utt[r] of `attended` [T',U,E]
 * (row_utt NULL = identity, U == R: the reference's replicated-context call).
 * states and next_states are [R, dec_stack * C]: with dec_stack 2 each row is [s0 | s1], the states of both layers
 * (the reference's "states" and "states#1").
 * `preprocessed` may be NULL: it is then recomputed, as the reference does on every call.
 * Content attention: the initial weights and energies are zeros (libs/blocks/blocks/bricks/attention.py:392-395), and
 * every energies output (here and in lvsr_cost_matrix) is zeros (lvsr/bricks/recognizer.py:475-478). */
int lvsr_initial_states(lvsr_model* m, int32_t Tp, int32_t R, float* states_dev, int64_t* outputs_dev,
                        float* weighted_averages_dev, float* weights_dev, float* energies_dev,
                        int64_t* step_dev, void* stream);
int lvsr_logprobs(lvsr_model* m, const float* attended_dev, const float* preprocessed_dev,
                  const float* attended_mask_dev, int32_t Tp, int32_t U, const int32_t* row_utt_dev,
                  int32_t R, const float* states_dev, const float* weights_dev, const int64_t* step_dev,
                  float* neg_logprobs_dev, void* stream);
/* lvsr_logprobs fused with the language model: lm_add_dev [R, V] is each row's LM cost row (lvsr_lm_initial_states /
 * lvsr_lm_next_states), and the output is the emitter cost -x of the fused readouts x, the row lvsr_beam_search_many
 * selects on.  lm_add_dev NULL: lvsr_logprobs.  lvsr_logprobs itself never fuses. */
int lvsr_logprobs_lm(lvsr_model* m, const float* attended_dev, const float* preprocessed_dev,
                     const float* attended_mask_dev, int32_t Tp, int32_t U, const int32_t* row_utt_dev,
                     int32_t R, const float* states_dev, const float* weights_dev, const int64_t* step_dev,
                     const float* lm_add_dev, float* neg_logprobs_dev, void* stream);
int lvsr_next_states(lvsr_model* m, const float* attended_dev, const float* preprocessed_dev,
                     const float* attended_mask_dev, int32_t Tp, int32_t U, const int32_t* row_utt_dev,
                     int32_t R, const float* states_dev, const float* weights_dev, const int64_t* step_dev,
                     const int64_t* outputs_dev, float* next_states_dev, float* next_weighted_averages_dev,
                     float* next_weights_dev, float* next_energies_dev, int64_t* next_step_dev,
                     void* stream);

/* ---- beam search: the whole loop of BeamSearch.search for MANY utterances -------------------------
 * (libs/blocks/blocks/search.py:244-399) for U utterances decoded in lock-step: all hypothesis state and the k-best
 * selection stay on the device, and the reference's bookkeeping (histories, `done`, both stopping criteria, final
 * ranking) runs in C++; per step one small H2D, one small D2H, one synchronisation for ALL utterances.
 * utt_len_host[u] = valid encoded frames, max_length_host[u] = int(T_u / max_decoded_length_scale)
 * (lvsr/bricks/recognizer.py:519-520).  stop_on_optimistic: 0 = 'patience', 1 = 'optimistic_future_cost'.
 * Result: per utterance the finished hypotheses ranked by cost - char_discount * length, each as its full token
 * and cumulative-cost history INCLUDING the initial symbol (what BeamSearch keeps in `done`).
 *
 * validate (may be NULL: every finished hypothesis is kept) is the reference's validate_solution_function
 * (:365-371): called once for every hypothesis that has just ended in eol_symbol, with the utterance index and
 * the full token history including the initial symbol, in utterance order and then in increasing candidate
 * order.  It returns 1 to add the hypothesis to `done`, 0 to drop it, and a negative value to abort the search:
 * lvsr_beam_search_many then returns non-zero without a result.  `validate_user` is passed through unchanged. */
typedef int32_t (*lvsr_validate_fn)(void* validate_user, int32_t utt, const int64_t* tokens, int32_t length);
typedef struct lvsr_search_result lvsr_search_result;
int lvsr_beam_search_many(lvsr_model* m, const float* attended_dev, const float* preprocessed_dev,
                          const float* attended_mask_dev, int32_t Tp, int32_t U, const int32_t* utt_len_host,
                          const int32_t* max_length_host, int32_t beam_size, int32_t eol_symbol,
                          int32_t ignore_first_eol, double char_discount, double round_to_inf,
                          int32_t stop_on_optimistic, lvsr_validate_fn validate, void* validate_user,
                          lvsr_search_result** result, void* stream);
int lvsr_search_result_count(const lvsr_search_result* r, int32_t utt);                     /* finished hypotheses */
int lvsr_search_result_length(const lvsr_search_result* r, int32_t utt, int32_t j);         /* history length     */
int lvsr_search_result_get(const lvsr_search_result* r, int32_t utt, int32_t j, int64_t* tokens, float* costs);
int lvsr_search_result_destroy(lvsr_search_result* r);

/* ---- FST language model, shallow fusion (lvsr/bricks/language_models.py, lvsr/ops.py:22-233) ----------------
 * lvsr_model_set_lm attaches an FST given as host arrays in NN label space: arcs of state s are
 * [arc_offsets[s], arc_offsets[s+1]) (arc_offsets has num_states + 1 entries), arc_label = NN symbol + 1 with
 * 0 = epsilon, each state's arcs sorted by (label, next state); arc weights are costs (negative log).  While it is
 * attached, lvsr_cost_matrix (and so lvsr_recognizer_cost_host) and lvsr_beam_search_many return the costs of
 * ShallowFusionReadout + LMEmitter instead of -log softmax (under task loss estimation: the loss of the fused readouts),
 * and lvsr_train_cost_and_grads refuses to run.
 * lvsr_cost_matrix then synchronises its stream once, to report an LM error.  lvsr_model_clear_lm detaches it.
 *
 * The LM state of a row is a set of at most LVSR_LM_MAX_STATES (fst state int32, weight float64) pairs padded with
 * state -1 / weight 0, and its cost row add [V] (float32; no_transition_cost where a symbol leads nowhere, and
 * everywhere once the set is empty).  lvsr_lm_initial_states writes expand({start: 0}) for R rows;
 * lvsr_lm_next_states advances row r by outputs[r] (int64).  Both synchronise the stream and return an error when a
 * set exceeds LVSR_LM_MAX_STATES, an epsilon closure exceeds 32 states or an epsilon cycle is met; the handle stays
 * usable. */
enum { LVSR_LM_MAX_STATES = 7 };
typedef struct {
  double weight;                   /* lm weight (reference default 0.0)                          */
  double am_beta;                  /* scale of the acoustic logits (1.0)                         */
  double no_transition_cost;       /* cost of a symbol without an arc (1e12)                     */
  int32_t normalize_am_weights;    /* log_softmax of the scaled logits (reference default 1)     */
  int32_t normalize_lm_weights;    /* log_softmax of -add (0)                                    */
  int32_t normalize_tot_weights;   /* log_softmax of the sum (0)                                 */
} lvsr_lm_fusion;
int lvsr_model_set_lm(lvsr_model* m, int32_t num_states, int32_t start, const int64_t* arc_offsets_host, int64_t num_arcs,
                      const int32_t* arc_label_host, const int32_t* arc_next_host, const float* arc_weight_host,
                      const lvsr_lm_fusion* fusion);
int lvsr_model_clear_lm(lvsr_model* m);
int lvsr_lm_initial_states(lvsr_model* m, int32_t R, int32_t* states_dev, double* weights_dev, float* add_dev,
                           void* stream);
int lvsr_lm_next_states(lvsr_model* m, int32_t R, const int32_t* states_dev, const double* weights_dev,
                        const int64_t* outputs_dev, int32_t* next_states_dev, double* next_weights_dev,
                        float* next_add_dev, void* stream);

/* ---- host-buffer entry points (the call a user of the reference makes) -------------
 * SpeechRecognizer.cost on a batch (lvsr/bricks/recognizer.py:375-390): H2D copies,
 * encoder, cost_matrix, D2H of costs [L,B]; synchronises.  Buffers should be pinned. */
int lvsr_recognizer_cost_host(lvsr_model* m, const float* recordings_host, const float* mask_host,
                              const int64_t* labels_host, const float* labels_mask_host,
                              int32_t T, int32_t B, int32_t L, float* costs_host, void* stream);

/* ---- training step: GradientDescent._function -------------------------------------------------
 * (libs/blocks/blocks/algorithms/__init__.py:244-256,284-287 as assembled by lvsr/main.py:340-345,480-519).
 * Split in two so a data-parallel caller can all-reduce the gradient buffer in between:
 *
 *   lvsr_train_cost_and_grads: forward + backward of one batch (device pointers, layouts as lvsr_encoder_forward /
 *     lvsr_cost_matrix).  cost_dev[0] = gscale * sum(cost_matrix); grads_dev (lvsr_model_flat_size floats, flat
 *     parameter layout) = gscale * d sum(cost_matrix) / d parameter.  Single GPU: gscale = 1/B gives the reference's
 *     cost = sum / batch_size.  N GPUs: pass gscale = 1, all-reduce(sum) grads_dev, then apply with
 *     gscale = 1 / global batch (SURVEY.md 8e).  A model with dec_stack 2 is refused before any work is enqueued
 *     (no backward pass through the stack).  Every energy normaliser: with logistic / relu the gradient of
 *     energy_comp/linear.b is formed too.  A relu row whose window holds no positive energy is 0 / 0 in the forward,
 *     as in the reference: its cost and the gradients are not finite (the update then follows RemoveNotFinite(0.0)).
 *   lvsr_train_apply_updates: grads_dev *= gscale (+ 2 decay W on WEIGHT parameters), then the CompositeRule of
 *     lvsr/main.py:509-516: StepClipping(gradient_threshold) -> Momentum(scale, momentum) -> AdaDelta(decay_rate,
 *     epsilon) -> Restrict(VariableClipping(max_norm, axis=0), WEIGHT parameters) -> RemoveNotFinite(0.0) -> BurnIn,
 *     parameter -= step, and the kernel-side weights are re-packed.  grads_dev holds the steps afterwards.
 *     Optimizer state lives in the handle (lvsr_train_reset clears it). */
typedef struct {
  float gradient_threshold;        /* StepClipping threshold, 0 = off (B/algorithms/__init__.py:610-643)        */
  int32_t use_momentum;            /* 'momentum' in config['training']['rules'] (lvsr/main.py:483-486)          */
  float scale, momentum;           /* Momentum(learning_rate=scale, momentum)                                   */
  int32_t use_adadelta;            /* 'adadelta' in rules                                                        */
  float decay_rate, epsilon;       /* AdaDelta(decay_rate, epsilon), :464-516                                    */
  float max_norm;                  /* regularization.max_norm, 0 = off (lvsr/main.py:490-505)                    */
  int32_t burn_in_steps;           /* BurnIn(num_steps), lvsr/algorithms.py:19-43                                */
  float decay;                     /* regularization.decay: + decay * ||WEIGHT parameters||^2 (lvsr/main.py:419-421) */
} lvsr_train_config;
int lvsr_train_cost_and_grads(lvsr_model* m, const float* recordings_dev, const float* mask_dev,
                              const int64_t* labels_dev, const float* labels_mask_dev, int32_t T, int32_t B,
                              int32_t L, float gscale, float* cost_dev, float* grads_dev, void* stream);
int lvsr_train_apply_updates(lvsr_model* m, float* grads_dev, float gscale, const lvsr_train_config* tc,
                             void* stream);
/* Under a task-loss criterion (lvsr_model_set_criterion) the cost lvsr_train_cost_and_grads differentiates is the
 * mse_gain / mse_reward rows of the labels scored against themselves: imitative exploration (lvsr/main.py:245-283).
 * Such a step synchronises its stream once, after all of its work is enqueued, to report a groundtruth that holds no
 * eos_label (naming the utterance; the gradient buffer is then undefined).
 * lvsr_train_cost_and_grads_greedy is the same step under greedy exploration (exploration: greedy):
 *   1. after the encoder, n = L + LVSR_GREEDY_EXTRA_STEPS steps of generate() on the device with the parameters the
 *      step runs on (under adaptive noise or weight noise, the noisy ones): prediction_dev [n, B] (int64) is the
 *      arg-max of the readouts at every step (the first on ties), from the state the previous pick fed;
 *   2. prediction_mask_dev [n, B] = 1 at step 0 and wherever no eos_label occurs in the earlier steps of the row;
 *   3. the step of lvsr_train_cost_and_grads on labels = the prediction, labels mask = its mask, with the rewards and
 *      gains of the prediction against groundtruth_dev [L, B] (every utterance of which must hold eos_label).
 * No gradient flows through the generation.  The groundtruth's mask plays no part: the prediction's own mask weights
 * the cost, as in the reference.  Refused: a log-likelihood handle; dropout and the alignment penalty, which the
 * reference leaves undefined under greedy exploration (its dropout graph holds two encoder applications, and its
 * penalty pairs n rows of alignments with the L-row label mask).  Detected by symbol. */
enum { LVSR_GREEDY_EXTRA_STEPS = 10 };
int lvsr_train_cost_and_grads_greedy(lvsr_model* m, const float* recordings_dev, const float* mask_dev,
                                     const int64_t* groundtruth_dev, int32_t T, int32_t B, int32_t L, float gscale,
                                     float* cost_dev, float* grads_dev, int64_t* prediction_dev,
                                     float* prediction_mask_dev, void* stream);
int lvsr_train_gradient_norm(lvsr_model* m, float* norm_host);   /* total_gradient_norm of the last update (synchronises
                                                                    the handle's stream) */
int lvsr_train_reset(lvsr_model* m);     /* zero the optimizer state, enqueued on the handle's stream after its updates */

/* ---- adaptive clipping: AdaptiveClipping (lvsr/extensions.py:64-91), which lvsr/main.py:616-619 always installs ----
 * While it is on, the StepClipping threshold of lvsr_train_apply_updates is the device value below, not
 * gradient_threshold.  After the norm of update n (n = 1, 2, ..., the float32 value lvsr_train_gradient_norm reports)
 * is reduced, the same kernel updates, in float64, with L = log(norm) and d = decay_rate:
 *   mu  <- d mu  + (1 - d) L          mu2 <- d mu2 + (1 - d) L^2          sigma = sqrt(mu2 - mu^2)
 *   c = min(burnin_period, n) / burnin_period
 *   threshold of update n + 1 = min(c exp(mu + sigma) + (1 - c) initial_threshold, 5 initial_threshold)
 * mu and mu2 start at 0 and update 1 clips with initial_threshold.  No launch, host copy or synchronisation is added
 * to the update; every data-parallel rank reduces the same all-reduced norm and so gets the same threshold.
 *   - a NaN norm makes the state and every later threshold NaN, as in the reference; a step clipped by a NaN threshold
 *     is NaN, so RemoveNotFinite(0.0) zeroes every parameter.
 *   - a zero norm (the reference raises on log(0)) leaves mu and mu2 unchanged; n still advances.
 *   - rounding that makes mu2 - mu^2 negative gives sigma = 0.
 * lvsr_train_set_adaptive_clipping turns it on (NULL: off) and resets the state; lvsr_train_reset resets it too.
 * lvsr_train_clipping_threshold returns the threshold the next update will use (synchronises the handle's stream;
 * an error while it is off). */
typedef struct {
  double initial_threshold;        /* thr_0: the StepClipping threshold (config['training']['gradient_threshold']) */
  double decay_rate;               /* d (lvsr/main.py: 0.998)                                                     */
  int32_t burnin_period;           /* (lvsr/main.py: 500)                                                          */
} lvsr_adaptive_clipping;
int lvsr_train_set_adaptive_clipping(lvsr_model* m, const lvsr_adaptive_clipping* cfg);
int lvsr_train_clipping_threshold(lvsr_model* m, double* threshold_host);

/* ---- adaptive weight noise (Graves 2011): apply_adaptive_noise, lvsr/graph.py:71-251, as lvsr/main.py:425-460
 * applies it to every parameter).  Each parameter p gets a log-variance ls2 of its shape, s2 = exp(2048 ls2).
 * While it is on:
 *   lvsr_train_cost_and_grads draws eps ~ N(0, 1) per element (Philox-4x32-10 keyed by (seed, update counter, flat
 *     index), Box-Muller in fp32: the same draw on every data-parallel rank), runs forward and backward on
 *     p + eps sqrt(s2), and computes from the means prior_u = mean(p), prior_s2 = mean(s2 + (p - prior_u)^2) and the
 *     model cost LC = coef / N * sum[0.5 (log prior_s2 - 2048 ls2) + ((p - prior_u)^2 + s2 - prior_s2) / (2 prior_s2)].
 *     Every other entry point sees the means and weights packed from them.  The cost it reports is the task cost.
 *   lvsr_train_apply_updates first forms, from g = gscale * grads_dev (the mean gradient at the noisy parameters),
 *     grad p = coef (p - prior_u) / (N prior_s2) + g and grad ls2 = coef 1024 / N (s2 / prior_s2 - 1) + 1024 s2 g^2,
 *     then runs the step rules over both groups: one clipping norm, optimizer state for both, RemoveNotFinite and
 *     BurnIn per tensor, max-norm on the WEIGHT means only.  It refuses decay > 0 (the reference takes the gradients
 *     of the cost without the decay term, lvsr/main.py:427-432).  The update counter then advances.  The weights
 *     are not re-packed from the new means: the next training forward packs its noisy copy, and any other entry
 *     point synchronises the device and packs the means first.
 * lvsr_train_set_adaptive_noise turns it on (NULL: off), sets every ls2 to log(init_sigma) / 1024, clears the ls2
 * optimizer state and the update counter.  lvsr_train_get/set_noise_param copy the ls2 of parameter `index`.
 * lvsr_train_noise_stats (synchronises): out[LVSR_NOISE_*] of the last training forward.
 * lvsr_train_noise_sample writes the eps of update `update` in the flat layout (padding zero).
 * lvsr_train_noise_params copies the noisy parameters the last training forward ran on (flat layout, padding zero).
 * lvsr_train_noise_gradients forms both gradient groups in place of grads_dev / into ls2_grads_dev (flat layout)
 *   without an update, with the priors of the last training forward. */
typedef struct {
  double init_sigma;               /* initial standard deviation of the noise (reference default 1e-6)          */
  double model_cost_coefficient;   /* coef (1.0)                                                                 */
  int64_t num_examples;            /* N: utterances in the training set                                          */
  uint64_t seed;                   /* key of the draw (the reference's default seed is 1)                         */
} lvsr_adaptive_noise;
enum { LVSR_NOISE_MODEL_COST = 0, LVSR_NOISE_PRIOR_MEAN = 1, LVSR_NOISE_PRIOR_VARIANCE = 2 };
int lvsr_train_set_adaptive_noise(lvsr_model* m, const lvsr_adaptive_noise* cfg);
int lvsr_train_get_noise_param(const lvsr_model* m, int index, float* values_host, int64_t count);
int lvsr_train_set_noise_param(lvsr_model* m, int index, const float* values_host, int64_t count);
int lvsr_train_noise_stats(lvsr_model* m, double out[3]);
int lvsr_train_noise_sample(lvsr_model* m, int64_t update, float* eps_dev, void* stream);
int lvsr_train_noise_params(lvsr_model* m, float* noisy_dev, void* stream);
int lvsr_train_noise_gradients(lvsr_model* m, float* grads_dev, float gscale, float* ls2_grads_dev, void* stream);

/* ---- dropout and weight noise: regularization.dropout / regularization.noise (lvsr/main.py:400-408) ----
 * While they are on, lvsr_train_cost_and_grads runs the step on regularised inputs; every other entry point
 * (cost, search, sampling, validation statistics) never applies them.
 *   dropout: the encoder's input (the recordings, or the bottom MLP's last output) is multiplied by Bernoulli(0.5) / 0.5
 *     element-wise, padded frames included (Blocks' apply_dropout).  The multiplier of element (t, b, f) is 0 or 2,
 *     drawn from Philox-4x32-10 keyed by (seed, update counter, global utterance index = utterance offset + b, t, f): a
 *     data-parallel rank given the offset of its first utterance draws the mask the one-GPU step on the concatenated
 *     batch draws.  The caller's recordings are not changed; with a bottom MLP its gradient passes the same multiplier.
 *   noise_level > 0: every parameter outside the attention brick (conv_att / cont_att) is perturbed by
 *     noise_level * eps, eps ~ N(0, 1) per element (Philox keyed by (seed, update counter, flat index), Box-Muller),
 *     for forward and backward (Blocks' apply_noise); the gradient at the noisy point is applied to the clean means,
 *     which decay and max-norm act on.  The attention's parameters are used as they are.
 * The update counter is advanced by lvsr_train_apply_updates and cleared by lvsr_train_reset and by
 * lvsr_train_set_regularization, so two lvsr_train_cost_and_grads calls between updates draw the same mask and noise.
 * Refused together with adaptive noise, under which the reference trains on the clean graph (lvsr/main.py:425-437).
 * lvsr_train_set_regularization sets them (NULL: both off); seed 0 means 1, Blocks' default seed.
 * lvsr_train_set_utterance_offset sets the global index of the batch's first utterance for the next steps (0 after
 *   lvsr_train_set_regularization).
 * lvsr_train_dropout_mask writes the multiplier of update `update` for a [T, B, F] batch whose first utterance has
 *   the global index `utterance_offset` (F: the encoder's input width).
 * lvsr_train_weight_noise_sample writes the eps of update `update` in the flat layout, exactly 0 in the padding and
 *   over the attention's parameters.
 * penalty_coof > 0: the alignment monotonicity penalty (lvsr/expressions.py:14-19) of the regularised forward's
 *   alignments w [L, B, T'], P = sum_b sum_{i>=1} m[i,b] sum_t max(c_i[t] - c_{i-1}[t], 0) with c_i = cumsum_t w_i and
 *   m the labels mask, adds penalty_coof * gscale * dP/dw to the alignment gradients (a tie c_i = c_{i-1} counts as
 *   increasing, as Theano's maximum does).  cost_dev stays the task cost; lvsr_train_penalty_sum copies P of the last
 *   training forward (a float, unscaled) to a device address on the stream, e.g. a slot of the all-reduced buffer. */
typedef struct {
  int32_t dropout;                 /* 1: dropout on the encoder's input, keep probability 0.5               */
  double noise_level;              /* standard deviation of the weight noise, 0 = off                        */
  double penalty_coof;             /* coefficient of the alignment penalty, 0 = off                          */
  uint64_t seed;                   /* key of both draws (0: 1)                                               */
} lvsr_regularization;
int lvsr_train_set_regularization(lvsr_model* m, const lvsr_regularization* cfg);
int lvsr_train_set_utterance_offset(lvsr_model* m, int64_t utterance_offset);
int lvsr_train_dropout_mask(lvsr_model* m, int64_t update, int64_t utterance_offset, int32_t T, int32_t B, int32_t F,
                            float* mult_dev, void* stream);
int lvsr_train_weight_noise_sample(lvsr_model* m, int64_t update, float* eps_dev, void* stream);
int lvsr_train_penalty_sum(lvsr_model* m, float* penalty_dev, void* stream);

/* ---- filterbank front end: Kaldi's compute-fbank-feats | add-deltas | global CMVN (exp/wsj/write_hdf_dataset.sh) ----
 * Waveforms in, the recognizer's recordings [T, B, D] and recordings_mask [T, B] out (DESIGN §1 (j) states the
 * definition).  Samples are float32 in int16 units, one mono utterance per row of a [B, row_stride] device buffer.
 * With W / S the frame length / shift in samples, an utterance of N >= W samples has 1 + (N - W) / S frames
 * (snip_edges); per frame: dither, DC removal, raw log energy, pre-emphasis, window, |real FFT|^2 of the frame
 * zero-padded to P (a power of two, at most LVSR_FBANK_MAX_PADDED), triangular mel banks, log; the row is
 * [log energy, bins] (use_energy) or [bins], D0 wide; delta_order > 0 appends the deltas of add-deltas
 * (D = D0 (delta_order + 1)); a global CMVN stats matrix, when given, normalises every column.
 *   - dither draws N(0, 1) per (utterance row, frame, sample of the frame) from Philox-4x32-10 keyed by seed, Box-Muller
 *     in fp32: a rerun with the same seed is bit-identical; lvsr_frontend_dither_sample writes the draws.
 *   - CMVN stats are Kaldi's [2, D + 1] float64 matrix: row 0 the column sums and the frame count in its last entry,
 *     row 1 the sums of squares.  Applying them: x' = (x - mean) / sqrt(max(s1 / n - mean^2, 1e-20)).
 *   - frames past an utterance's end (up to T) are exactly 0 with mask 0.
 * lvsr_frontend_create refuses, before any device work, snip_edges 0, vtln_warp != 1, htk_compat 1, use_log_fbank 0,
 * a frame longer than LVSR_FBANK_MAX_PADDED samples and options outside Kaldi's ranges; lvsr_frontend_compute
 * refuses an utterance shorter than one frame, naming its row.  The handle is bound to the device current at create,
 * and to streams as the model handle is (the stream rule at the top of this file); it owns its tables and workspace.
 * Added within version 104: detect these calls by their symbols. */
enum { LVSR_WINDOW_POVEY = 0, LVSR_WINDOW_HAMMING = 1, LVSR_WINDOW_HANNING = 2, LVSR_WINDOW_RECTANGULAR = 3 };
enum { LVSR_FBANK_MAX_PADDED = 512, LVSR_FBANK_MAX_DELTA_ORDER = 3, LVSR_FBANK_MAX_DELTA_WINDOW = 4 };
typedef struct {                     /* Kaldi's option names; (the recipes' values)                                  */
  double sample_frequency;           /* Hz (16000)                                                                   */
  double frame_length;               /* ms (25)                                                                      */
  double frame_shift;                /* ms (10)                                                                      */
  double dither;                     /* standard deviation of the dither, int16 units (1.0); 0 = off                 */
  double preemphasis_coefficient;    /* (0.97)                                                                       */
  double low_freq;                   /* Hz, lower edge of the mel banks (20)                                         */
  double high_freq;                  /* Hz, upper edge; <= 0: Nyquist + high_freq (0)                                */
  double energy_floor;               /* > 0: log energy floored at log(energy_floor) (0)                             */
  double vtln_warp;                  /* must be 1 (no VTLN)                                                          */
  uint64_t seed;                     /* key of the dither draws                                                      */
  int32_t remove_dc_offset;          /* (1)                                                                          */
  int32_t window_type;               /* LVSR_WINDOW_* (povey)                                                        */
  int32_t round_to_power_of_two;     /* (1); 0 only for a frame of a power-of-two length                             */
  int32_t snip_edges;                /* must be 1                                                                    */
  int32_t num_mel_bins;              /* (40)                                                                         */
  int32_t use_energy;                /* (1)                                                                          */
  int32_t raw_energy;                /* 1: energy before pre-emphasis and window (1)                                 */
  int32_t use_log_fbank;             /* must be 1                                                                    */
  int32_t use_power;                 /* 1: power spectrum, 0: magnitude (1)                                          */
  int32_t htk_compat;                /* must be 0                                                                    */
  int32_t delta_order;               /* add-deltas --delta-order, 0 .. LVSR_FBANK_MAX_DELTA_ORDER (2)                */
  int32_t delta_window;              /* add-deltas --delta-window, 1 .. LVSR_FBANK_MAX_DELTA_WINDOW (2)              */
} lvsr_fbank_options;
typedef struct lvsr_frontend lvsr_frontend;
int lvsr_frontend_create(const lvsr_fbank_options* opts, lvsr_frontend** out);
int lvsr_frontend_destroy(lvsr_frontend* f);
/* frames of an utterance of num_samples samples (0 when shorter than one frame); -1 on a null handle */
int64_t lvsr_frontend_num_frames(const lvsr_frontend* f, int64_t num_samples);
/* D, the width of a feature row; -1 on a null handle */
int lvsr_frontend_feature_dim(const lvsr_frontend* f);
/* samples_dev [B, row_stride] float32 (16-byte aligned, row_stride a multiple of 4), lengths_host[b] <= row_stride the
 * samples of row b; T >= every row's frame count.  Writes features_dev [T, B, D] and mask_dev [T, B] (float 0 / 1).
 * cmvn_stats_dev: [2, D + 1] float64 on the device, or NULL for no CMVN. */
int lvsr_frontend_compute(lvsr_frontend* f, const float* samples_dev, int64_t row_stride, const int64_t* lengths_host,
                          int32_t B, int32_t T, float* features_dev, float* mask_dev, const double* cmvn_stats_dev,
                          void* stream);
/* Adds the sums of the frames of features_dev [T, B, D] whose mask_dev [T, B] entry is > 0.5 (NULL: every frame) to
 * stats_dev [2, D + 1] float64: per-CTA float64 partial sums over fixed row ranges, reduced in a fixed order, so
 * the result depends on the batch alone. */
int lvsr_frontend_accumulate_cmvn(lvsr_frontend* f, const float* features_dev, const float* mask_dev, int32_t T,
                                  int32_t B, double* stats_dev, void* stream);
/* Normalises features_dev [T, B, D] in place by stats_dev, on the frames whose mask is > 0.5 (NULL: every frame). */
int lvsr_frontend_apply_cmvn(lvsr_frontend* f, float* features_dev, const float* mask_dev, int32_t T, int32_t B,
                             const double* stats_dev, void* stream);
/* The dither's N(0, 1) draws for utterance rows 0 .. B-1 and frames 0 .. T-1: draws_dev [B, T, W] (unscaled). */
int lvsr_frontend_dither_sample(lvsr_frontend* f, int32_t B, int32_t T, float* draws_dev, void* stream);

/* Counters for bench.py: number of kernels this library launched since the last reset. */
int64_t lvsr_launch_count(int reset);
/* Bytes of device memory the library's model and front-end handles hold (their workspaces included), process-wide. */
int64_t lvsr_device_bytes(void);

/* Per-kernel-class device timing (CUDA events recorded on the launching stream around every
 * launch of that class) -- the analogue of the reference's Theano ProfileStats
 * (libs/Theano/theano/compile/profiling.py:97).  Classes: "gemm", "bigru", "attention",
 * "window", "dense", "readout", "lm", "noise" (adaptive weight noise), "bottom" (the bottom MLP's forward, its
 * GEMMs included), "bottom_bwd" (its backward), "dropout" (the training dropout's forward and backward) and
 * "weight_noise" (the sample of regularization.noise) and "penalty" (the alignment penalty's gradient and sum) and
 * "fbank" (the two kernels of lvsr_frontend_compute).  lvsr_profile_read synchronises the device, returns the
 * summed milliseconds and launch count recorded since the last read of that class. */
int lvsr_profile_enable(int on);
int lvsr_profile_read(const char* kernel_class, double* total_ms, int64_t* count);

#ifdef __cplusplus
}
#endif
#endif /* LVSR_B200_H */
