/*
 * seist_b200 — C-ABI of the CUDA-native SeisT forward/backward hot path.
 *
 * The reference (senli1073/SeisT) is pure Python/PyTorch and has no FFI of its own; the interfaces
 * these entry points replace are the torch.nn leaf modules its model calls
 * (models/seist.py) — cited per op kind below — plus models/loss.py:32-56 (BCELoss),
 * torch.nn.HuberLoss (models/loss.py:3) and the Adam step of training/train.py:304-308,109-111.
 *
 * Conventions: plain pointers and sizes only (no torch types); every pointer is a DEVICE pointer
 * into memory owned by the caller (torch-allocated); all tensors are contiguous fp32 (N, C, L)
 * ("NCL", sample axis contiguous) unless stated; every call is asynchronous on `stream`
 * (a cudaStream_t passed as void*), never allocates, never synchronises and is CUDA-graph
 * capturable.  Return value: 0 ok, <0 argument error, >0 cudaError_t.
 *
 * The network is executed as a *plan*: an array of SeistOp descriptors built once by the host
 * (seist_b200/plan.py) and run by seist_plan_run().  A descriptor names its operands as *views*:
 * a (channel-slice of a) materialised pre-BatchNorm tensor plus the BatchNorm / activation that
 * the consumer applies on load.  BatchNorm statistics are accumulated by the producer's epilogue
 * into the BN table, so a training-mode BN never costs its own pass over memory.
 */
#ifndef SEIST_B200_H_
#define SEIST_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SEIST_ABI_VERSION 24
#define SEIST_MAX_IN 3

/* ---- BatchNorm table entry (nn.BatchNorm1d, models/seist.py:641; SURVEY §3.5) ---------------- */
typedef struct SeistBN {
  const float* gamma;    /* [C] weight */
  const float* beta;     /* [C] bias */
  float* running_mean;   /* [C] */
  float* running_var;    /* [C] */
  double* stat;          /* [2C] sum(x), sum(x^2) of the BN input over (N, L)  (all ranks)       */
  double* gstat;         /* [2C] sum(du), sum(du * khat) of the gradient w.r.t. the BN output     */
  double* stat_acc;      /* where the producers' epilogues ACCUMULATE this rank's part of `stat`: the same
                            buffer on one GPU; under data parallelism (SyncBatchNorm, reference
                            training/train.py:374) a buffer in NVLink-symmetric memory that the
                            BN_PREPARE exchange sums over all ranks into `stat`                  */
  double* gstat_acc;     /* idem for `gstat`                                                      */
  float* dgamma;         /* [C] */
  float* dbeta;          /* [C] */
  float* coef;           /* [C][8] per-channel coefficients written by the BN_PREPARE ops:
                            0 scale, 1 shift (BN(x) = scale*x + shift, chained BN folded in),
                            2 mu, 3 istd (khat = (x-mu)*istd), 4 A, 5 Bx, 6 Cc (dx = A*du + Bx*x + Cc)  */
  double count;          /* elements per channel behind `stat` (global batch * L)                 */
  int32_t C;
  int32_t chain;         /* index of a second BN applied directly on top (attention.norm after
                            aggr.norm, models/seist.py:95,374) or -1                              */
  int32_t use_batch;     /* 1 train (batch statistics), 0 eval (running statistics)               */
  int32_t is_chained;    /* 1: this entry is the *second* BN of a chain (statistics derived)      */
  float eps;
  float momentum;
  float grad_scale;      /* multiplies dgamma/dbeta (1/world_size under data parallelism)         */
} SeistBN;

/* ---- data-parallel exchange over NVLink peer memory (replaces the per-BatchNorm NCCL calls of
   torch.nn.SyncBatchNorm, torch/nn/modules/_functions.py, enabled by reference training/train.py:374,
   and the DDP gradient all-reduce of training/train.py:369): every rank maps every other rank's
   buffers (torch.distributed._symmetric_memory / cuMem fabric handles) and the kernels read them
   directly; a per-lane epoch counter + release/acquire signal words form the barrier. -------------- */
#define SEIST_MAX_WORLD 8
#define SEIST_SIG_LANES 4   /* 0 forward statistics, 1 backward statistics, 2 gradients ready, 3 gradients consumed */
typedef struct SeistComm {
  int32_t world, rank;
  double* stat_peer[SEIST_MAX_WORLD];   /* base of rank p's stat_acc buffer (peer-mapped device pointers)       */
  double* gstat_peer[SEIST_MAX_WORLD];  /* base of rank p's gstat_acc buffer                                    */
  float* grad_peer[SEIST_MAX_WORLD];    /* base of rank p's flat gradient buffer                                */
  uint32_t* sig_peer[SEIST_MAX_WORLD];  /* rank p's signal pad: uint32 [SEIST_SIG_LANES][SEIST_MAX_WORLD]        */
  uint32_t* epoch;                      /* local uint32 [SEIST_SIG_LANES]: exchanges issued per lane             */
  int32_t* err;                         /* local: set to 1 when a peer wait timed out (bounded spin)            */
} SeistComm;

/* ---- operand view ---------------------------------------------------------------------------- */
typedef struct SeistView {
  float* x;        /* base of the (N, Ct, L) tensor                                               */
  float* g;        /* gradient buffer, same geometry: w.r.t. BN(x) if bn>=0 else w.r.t. x; or NULL */
  int32_t Ct;      /* channels of the underlying buffer                                           */
  int32_t c0;      /* first channel of the slice                                                  */
  int32_t C;       /* channels in the slice (0 = view absent)                                     */
  int32_t L;       /* samples                                                                     */
  int32_t bn;      /* BN table index applied on load, -1 none                                     */
  int32_t bn_c0;   /* channel offset of the slice inside that BN                                  */
  int32_t act;     /* 0 none, 1 exact-erf GELU (models/seist.py:640)                              */
  int32_t accum;   /* backward: 0 overwrite g, 1 add into g                                       */
} SeistView;

enum SeistOpKind {
  /* generalised 1-D convolution: out = alpha(n)*[drop(conv(f(in)) + bias) + res_a] + res_b.
     Covers nn.Conv1d k=1 (models/seist.py:86,107,111,130,142,182,225,287,351-364,429,451),
     depthwise (:134-141), grouped (:215-222) and dense head convs (:536,546) with _auto_pad_1d
     (:12-48); the input may be avg+max pooled (:80-81,93) or linearly up-sampled (:566);
     channel concat (:192,315,500) is a multi-view input or a channel-sliced output;
     Dropout/DropPath (:114,228,239,360-366,446,470,484) are the drop()/alpha() factors. */
  SEIST_OP_CONV_FWD = 1,
  SEIST_OP_CONV_BWD_DATA = 2,   /* gradient to the input views                                    */
  SEIST_OP_CONV_BWD_W = 3,      /* dW, dbias                                                      */
  SEIST_OP_RES_BWD = 4,         /* gradient to res_a / res_b                                      */
  /* AttentionBlock core softmax((q/sqrt(E))^T k) v^T, models/seist.py:381-388 */
  SEIST_OP_ATT_FWD = 5,
  SEIST_OP_ATT_BWD_Q = 6,
  SEIST_OP_ATT_BWD_KV = 7,
  /* HeadRegression / HeadClassification: mean over L -> Linear -> act, models/seist.py:575-610 */
  SEIST_OP_HEADVEC_FWD = 8,
  SEIST_OP_HEADVEC_BWD = 9,
  /* running-stat update / dgamma,dbeta for every BN of the table in one launch */
  SEIST_OP_BN_FINALIZE_FWD = 10,
  SEIST_OP_BN_FINALIZE_BWD = 11,
  SEIST_OP_ZERO = 12,           /* memset out.x[0 .. zero_bytes)                                   */
  /* per-channel coefficient tables of BN entries [bn_lo, bn_lo + n_bn): forward (scale, shift, mu,
     istd) once the statistics are complete; backward (A, Bx, Cc) once gstat is complete */
  SEIST_OP_BN_PREPARE_FWD = 13,
  SEIST_OP_BN_PREPARE_BWD = 14,
  /* DSConvNormAct (models/seist.py:124-155) is linear up to its BatchNorm: in_proj (1x1, no bias),
     zero pad, depthwise k-tap, pconv (1x1, no bias) compose into ONE dense k-tap convolution
       W_eff[o][i][t] = sum_c pconv[o][c] * dconv[c][t] * in_proj[c][i]
     so the two intermediate tensors of every stem path never exist.  COMPOSE_FWD writes W_eff
     (out.x) from in[0].x = in_proj [C,C], in[1].x = dconv [C,k], in[2].x = pconv [Cout,C];
     COMPOSE_BWD scatters dW_eff (out.g) into in[0..2].g. */
  SEIST_OP_STEM_COMPOSE_FWD = 15,
  SEIST_OP_STEM_COMPOSE_BWD = 16
};

typedef struct SeistOp {
  int32_t kind;
  int32_t N;                    /* local batch */
  const SeistBN* bn_table;      /* device copy of the BN table */
  const uint64_t* step_seed;    /* device scalar mixed into every dropout stream (may be NULL)     */

  SeistView in[SEIST_MAX_IN];   /* channel-concatenated inputs (ATT: q, k, v)                      */
  SeistView res_a;
  SeistView res_b;
  SeistView out;                /* out.bn/bn_c0: BN whose statistics the epilogue accumulates;
                                   out.g: gradient w.r.t. BN(out) (backward)                       */
  float* out_dxd;               /* gradient w.r.t. out directly (backward), or NULL                */

  const float* W;               /* [Cout, Cin/groups, k]                                           */
  const float* bias;            /* [Cout] or NULL                                                  */
  float* dW;
  float* dbias;

  int32_t n_in;
  int32_t Cin;                  /* sum of in[].C                                                   */
  int32_t Cout;
  int32_t k;
  int32_t stride;
  int32_t pad_left;
  int32_t groups;
  int32_t pool;                 /* >1: input is AvgPool1d(pool,ceil)+MaxPool1d(pool,ceil) of the view */
  int32_t up_src_L;             /* >0: input is F.interpolate(linear) of a view of this length      */
  int32_t L_in;                 /* conv-input length (after pool / upsample, before padding)        */
  int32_t L_out;
  int32_t out_act;              /* 0 none, 1 sigmoid, 2 softmax (HEADVEC only)                      */
  float out_scale;              /* HEADVEC: ScaledActivation factor                                 */

  float p_elem;                 /* nn.Dropout on conv(...)+bias                                     */
  float p_path;                 /* DropPath on the same quantity (per sample)                       */
  float p_alpha;                /* outer DropPath alpha(n) (MPTL gconv_droppath)                    */
  uint32_t seed_elem;
  uint32_t seed_path;
  uint32_t seed_alpha;

  /* attention */
  float* lse;                   /* [N, heads, Lq] log-sum-exp saved by the forward                  */
  float* delta;                 /* [N, heads, Lq] scratch for the backward                          */
  int32_t heads;
  float p_attn;
  uint32_t seed_attn;
  int32_t pad0_;

  const SeistComm* comm;        /* BN_PREPARE: device copy of the exchange descriptor, NULL on one GPU              */
  uint64_t zero_bytes;          /* SEIST_OP_ZERO */
  int32_t n_bn;                 /* BN_FINALIZE: entries in bn_table; BN_PREPARE: entries to prepare */
  int32_t bn_lo;                /* BN_PREPARE: first entry                                          */
  /* lane schedule (seist_plan_run_lanes; seist_b200/schedule.py): the stream this op is issued on, the events
     (recorded by earlier ops of OTHER lanes) it waits for first, the event it records when done (-1 none) */
  int32_t lane;
  int32_t n_wait;
  int32_t wait_ev[4];
  int32_t rec_event;
  int32_t pad1_;
} SeistOp;

/* ---- entry points ---------------------------------------------------------------------------- */
int seist_abi_version(void);
uint64_t seist_sizeof_op(void);
uint64_t seist_sizeof_bn(void);
const char* seist_last_error(void);
/* number of kernel launches issued by this library since load (bench `gpu_launches`) */
uint64_t seist_launch_count(void);
/* name of the kernel family the dispatcher launches for `op` (e.g. "pw_fwd(simt)"); static string */
const char* seist_op_family(const SeistOp* op);
/* 1 if a tensor-core kernel ever timed out waiting on one of its mbarriers (bounded spin) */
int seist_tc_error_flag(void);

/* run ops[0..n) in order on `stream` */
int seist_plan_run(const SeistOp* ops, int32_t n, void* stream);

/* run ops[0..n) on `n_streams` streams by the lane schedule stored in the descriptors: op i is issued on
   streams[min(lane, n_streams-1)] after waiting for its `wait_ev` events; all lanes are forked from streams[0] at the start
   and joined back into it at the end (CUDA-graph capturable: the events become graph edges).  */
int seist_plan_run_lanes(const SeistOp* ops, int32_t n, void* const* streams, int32_t n_streams);

/* BCELoss(weight) with eps inside the logs — models/loss.py:48-56.  preds/targets (N,C,L);
   weight [C]; loss_sum: device double accumulator (zeroed by the call); *loss_out = sum / numel. */
int seist_bce_fwd(const float* preds, const float* targets, const float* weight, int64_t N, int32_t C,
                  int64_t L, float eps, double* loss_sum, float* loss_out, void* stream);
/* dpreds = gout * dloss/dpreds  (gout: device scalar, upstream gradient of the mean loss) */
int seist_bce_bwd(const float* preds, const float* targets, const float* weight, const float* gout,
                  int64_t N, int32_t C, int64_t L, float eps, float* dpreds, void* stream);
/* CELoss(weight) on class probabilities (N, C): mean_n sum_c -w[c] t[n,c] log(p[n,c] + eps) - models/loss.py:8-29,
   the loss of the seist_*_pmp variants (config.py:147-155) */
int seist_ce_fwd(const float* preds, const float* targets, const float* weight, int64_t rows, int32_t C, float eps,
                 double* loss_sum, float* loss_out, void* stream);
int seist_ce_bwd(const float* preds, const float* targets, const float* weight, const float* gout, int64_t rows,
                 int32_t C, float eps, float* dpreds, void* stream);
/* torch.nn.HuberLoss(delta) mean — models/loss.py:3, config.py:158 */
int seist_huber_fwd(const float* preds, const float* targets, int64_t numel, float delta,
                    double* loss_sum, float* loss_out, void* stream);
int seist_huber_bwd(const float* preds, const float* targets, const float* gout, int64_t numel,
                    float delta, float* dpreds, void* stream);

/* torch.optim.Adam / AdamW (decoupled=1) single fused update over one flat buffer —
   training/train.py:304-316.  lr and step are device scalars so the call is graph-replayable; the
   hyper-parameters are doubles like torch's python floats ((1 - beta) is formed in double). */
int seist_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t numel,
                    const float* lr, const float* step, double beta1, double beta2, double eps,
                    double weight_decay, int32_t decoupled, float grad_scale, void* stream);
/* torch.optim.SGD(momentum, dampening, weight_decay, nesterov) single fused update over one flat buffer —
   training/train.py:316-322.  d = grad_scale * g (+ weight_decay * p); with momentum != 0 the buffer is d on the
   first step and momentum * buf + (1 - dampening) * d after it, and d becomes buf (or d + momentum * buf with
   nesterov); p -= lr * d.  The first step is *step <= 1 on the device (the caller increments step before the call),
   so the call is graph-replayable.  momentum_buf may be NULL when momentum == 0; nesterov needs momentum > 0 and
   dampening == 0. */
int seist_sgd_step(float* params, const float* grads, float* momentum_buf, int64_t numel, const float* lr,
                   const float* step, double momentum, double dampening, double weight_decay, int32_t nesterov,
                   float grad_scale, void* stream);

/* Gradient all-reduce (sum) over peer memory: out[i] = sum_p grad_peer[p][i], bracketed by two cross-rank
   barriers (all gradients complete / all peers finished reading).  `comm` is the DEVICE copy; graph capturable. */
int seist_comm_allreduce(const SeistComm* comm, int32_t world, float* out, int64_t numel, void* stream);
/* cross-rank barrier on signal lane `lane` (tests / teardown) */
int seist_comm_barrier(const SeistComm* comm, int32_t lane, void* stream);
uint64_t seist_sizeof_comm(void);

/* ---- post-processing on the device (SURVEY 8f-1; reference training/postprocess.py, utils/metrics.py) -----------
   prob: (N, C, L) fp32 probabilities (the dpk head's output); `channel` selects the trace.
   seist_pick_phase   = _pick_phase (postprocess.py:161-193 -> _detect_peaks :15-111, rising edges, mph = threshold,
                        mpd = min_peak_dist > 1, topk): out (N, topk) int64 sample indices, padded with pad_value.
   seist_detect_event = _detect_event (:114-158 -> obspy trigger_onset(x, thr, thr)): out (N, 2*topk) int64 [on, off]
                        pairs of the topk longest runs of prob > thr, padded with [1, 0].
   seist_pick_counters / seist_det_counters = the tp / predp / possp (+ residual sums) of utils/metrics.py:141-232,
                        ADDED into a double vector `acc` (pick: 7 entries, det: 4) so that several tasks and steps share
                        one buffer and one all-reduce.  Integer results are bit-identical to oracle/postprocess_ref.py. */
int seist_pick_phase(const float* prob, int64_t N, int32_t C, int32_t channel, int32_t L, float threshold,
                     int32_t min_peak_dist, int32_t topk, int64_t pad_value, int64_t* out, void* stream);
int seist_detect_event(const float* prob, int64_t N, int32_t C, int32_t channel, int32_t L, float threshold,
                       int32_t topk, int64_t* out, void* stream);
int seist_pick_counters(const int64_t* targets, const int64_t* preds, int64_t n, int32_t num_samples, int32_t t_thres,
                        double* acc, void* stream);
int seist_det_counters(const int64_t* targets, const int64_t* preds, int64_t N, int32_t k_targets, int32_t k_preds,
                       int32_t num_samples, double* acc, void* stream);

/* ---- input side on the device (SURVEY 8f-3; reference training/preprocess.py) ---------------------------------------
   seist_normalize  = DataPreprocessor._normalize (:224-242) over `rows` traces of L samples, in place: mean removal,
                      then mode 1 "std" / 2 "max" scaling (a zero scale is replaced by 1), mode 0 "" mean removal only.
   seist_dpk_labels = the label stack [det, ppk, spk] of the dpk task (config.py:137-146) from the phase indices:
                      _generate_soft_label (:544-683) with _pad_phases (:16-35).  ppks / spks: (N, K) int64, entries
                      <= -1000000 mean "no phase"; shape 0 gaussian (sigma 10 samples) / 1 triangle / 2 box /
                      3 sigmoid (width >= 2); out (N,3,L). */
int seist_normalize(float* x, int64_t rows, int32_t L, int32_t mode, void* stream);
int seist_dpk_labels(const int64_t* ppks, const int64_t* spks, int64_t N, int32_t K, int32_t L, int32_t width,
                     int32_t shape, double coda_ratio, float* out, void* stream);

/* ---- training-time augmentation on the device (reference training/preprocess.py) ---------------------------------
   seist_augment = DataPreprocessor.process (:501-542) for a batch: _is_noise, _pad_phases, _data_augmentation (:432-499)
                   where augment[n] != 0 (every trace when augment is NULL), _cut_window (:172-222), _normalize.
                   data (N, C, Lin) fp32, 3 <= Lin <= 16384 and C * Lin * 4 bytes within the shared memory of one CTA;
                   ppks / spks (N, K) int64, entries <= -1000000 mean "no phase"; snr (N, S) double or S = 0.
                   Writes x (N, C, cfg->in_samples), the output phase lists ppks_out / spks_out (N, K_out) padded with
                   -10000000, cleared (N,) (1 where _is_noise or the generated noise cleared the event).  Draws come from a
                   counter-based generator at *seed (device scalar, not advanced here).  work: N * seist_aug_recipe_bytes().
   seist_sizeof_aug = sizeof(SeistAugCfg), for the binding's layout check. */
typedef struct SeistAugCfg {
  double generate_noise_rate, add_event_rate, shift_event_rate, drop_channel_rate, scale_amplitude_rate;
  double pre_emphasis_rate, add_noise_rate, add_gap_rate;
  double coda_ratio, min_snr, p_position_ratio;  /* p_position_ratio in [0, 1]: deterministic cut with P at that ratio */
  float pre_emphasis_ratio;
  int32_t in_samples, min_event_gap;             /* min_event_gap in samples */
  int32_t max_event_num, norm_mode;              /* norm_mode 0 "", 1 "std", 2 "max" */
  int32_t mask_percent, noise_percent, window;   /* window = sampling_rate // 2 samples, at most 1024 windows per trace */
} SeistAugCfg;
uint64_t seist_sizeof_aug(void);
int seist_aug_recipe_bytes(void);
int seist_augment(const float* data, int64_t N, int32_t C, int32_t Lin, const int64_t* ppks, const int64_t* spks, int32_t K,
                  const double* snr, int32_t S, const uint8_t* augment, const SeistAugCfg* cfg, const uint64_t* seed,
                  float* x, int64_t* ppks_out, int64_t* spks_out, int32_t K_out, uint8_t* cleared, void* work,
                  int64_t work_bytes, void* stream);

/* ---- continuous records (DESIGN §4.15): sliding-window inference, overlap stacking, whole-record picking ------------
   The reference runs one window (demo_predict.py:75 keeps record[:, :8192]); these restate, per window of W samples at
   stride P, `_normalize` (training/preprocess.py:224-242), and on the stacked traces `_detect_peaks` with topk = None
   (training/postprocess.py:15-111) and obspy trigger_onset(p, thr, thr) (:114-158) with every run kept.
   Windows of a station: starts k * P for k = 0 .. (T - W) / P, plus T - W when the last of those ends before T; K per
   station, window id s * K + k.  record (S, C, T) and probs (S, 3, T) fp32, W <= T < 2^31, 1 <= P <= W.
   seist_window_batch  = the (B, C, W) model input of windows w0 .. w0 + B - 1, each row normalised as seist_normalize
                         (mode 0 none, 1 std, 2 max; W <= 49152); ids >= S * K give zero rows.
   seist_stack_batch   = adds (mode 0) or fmaxf's (mode 1) the (B, 3, W) outputs of windows w0 .. w0 + B - 1 into probs;
                         each sample takes its covering windows in ascending id order, starting from 0.0f / -inf at its
                         first covering window.  Call with w0 = 0, B, 2B, ... in order on one stream.
   seist_stack_finish  = mode 0: probs /= number of covering windows (one IEEE division).
   seist_peaks_long    = `_detect_peaks(probs[s, channel], mph, mpd > 1, topk=None)` of every row (rising edges, equal
                         heights: the larger index ranks first); writes counts (S,) int64 and keeps its state in `work`
                         (seist_peaks_work_bytes).  seist_peaks_long_fill then writes the picks of row s, in index order, at
                         index / value[offsets[s] ..] (offsets: exclusive prefix sums of counts, int64).
   seist_runs_long     = the inclusive [on, off] of every maximal run of probs[s, channel] > threshold, in time order:
                         counts (S,) int64; seist_runs_long_fill writes pairs[offsets[s] ..] (E, 2) int64.
   The two passes of each pick / run call share `work` and must see the same prob. */
int seist_window_batch(const float* record, int32_t S, int32_t C, int64_t T, int32_t W, int32_t P, int64_t w0, int32_t B,
                       int32_t mode, float* x, void* stream);
int seist_stack_batch(const float* y, int32_t S, int64_t T, int32_t W, int32_t P, int64_t w0, int32_t B, int32_t mode,
                      float* probs, void* stream);
int seist_stack_finish(float* probs, int32_t S, int64_t T, int32_t W, int32_t P, void* stream);
int64_t seist_peaks_work_bytes(int32_t S, int64_t T);
int seist_peaks_long(const float* prob, int32_t S, int32_t C, int32_t channel, int64_t T, float mph, int32_t min_peak_dist,
                     void* work, int64_t work_bytes, int64_t* counts, void* stream);
int seist_peaks_long_fill(int32_t S, int64_t T, const void* work, int64_t work_bytes, const int64_t* offsets, int64_t* index,
                          float* value, void* stream);
int64_t seist_runs_work_bytes(int32_t S, int64_t T);
int seist_runs_long(const float* prob, int32_t S, int32_t C, int32_t channel, int64_t T, float threshold, void* work,
                    int64_t work_bytes, int64_t* counts, void* stream);
int seist_runs_long_fill(const float* prob, int32_t S, int32_t C, int32_t channel, int64_t T, float threshold, const void* work,
                         int64_t work_bytes, const int64_t* offsets, int64_t* pairs, void* stream);

/* ---- picked events on continuous records (DESIGN §4.17): P-anchored windows for the non-dpk heads -------------------
   The reference cuts one event window with `_cut_window` and 0 <= p_position_ratio <= 1 (training/preprocess.py:172-203):
   W samples with the first P pick at sample anchor = int(W * p_position_ratio) (computed by the caller), zero-filled
   outside the trace, then `_normalize` (:224-242).  record (S, C, T) fp32, 1 <= T < 2^31; index (M,) int64 P sample
   indices (may be null when M = 0) and offsets (S + 1,) int64 the CSR of seist_peaks_long_fill (station s holds events offsets[s] .. offsets[s+1]).
   seist_event_windows = for d < n_dst (<= 4), x[d] (B, C, W) = the input of events e0 .. e0 + B - 1: row (b, c) is
                         record[s, c, p - anchor + i], i < W, with 0.0f outside [0, T), normalised as seist_normalize (mode
                         0 none, 1 std, 2 max; W <= 49152); p = index[e0 + b], s the last station with offsets[s] <= e0 + b
                         (a bounded search: always in [0, S)).  Events >= M and picks outside [0, T) give zero rows (the
                         reference's slicing would wrap around there).  Offsets are never read back to the host. */
int seist_event_windows(const float* record, int32_t S, int32_t C, int64_t T, const int64_t* index, int64_t M,
                        const int64_t* offsets, int64_t e0, int32_t B, int32_t W, int32_t anchor, int32_t mode, float* const* x,
                        int32_t n_dst, void* stream);

/* ---- continuous records streamed chunk by chunk (DESIGN §4.16) -------------------------------------------------------
   One call of a stream (a push of n samples per station, or the close) as global int64 sample counts from the start of the
   stream.  Before the call R = r0 samples were pushed and the samples [0, f0) were emitted; after it R = r1 and [0, f1) are
   final (f = max(0, R - W) before the close, T at the close).  The call runs the regular windows k0 .. k0 + nk - 1 of every
   station (start k * P) and, at the close, the tail window starting at `tail` (-1: none); kr is the record's number of
   regular windows at the close and -1 before.  The call's window j is window j % (nk + (tail >= 0)) of station
   j / (nk + (tail >= 0)), the tail one last.  Buffers (row-major, fp32):
     tail_raw  (S, C, W): the last min(W, r0) raw samples, [r0 - min(W, r0), r0); tail_out the same after the call.
     chunk     (S, C, n = r1 - r0).
     carry     (S, 3, W): partial sums of [f0, r0); carry_out (S, 3, W) those of [f1, r1) after the call.
     acc       (S, 3, r1 - f0): the call's partial sums of [f0, r1).
     probs     (S, 3, f1 - f0): the final probabilities of [f0, f1).
   seist_stream_window = seist_window_batch for the call's windows j0 .. j0 + B - 1, cut from tail_raw ++ chunk.
   seist_stream_stack  = seist_stack_batch of those windows' outputs y (B, 3, W) into acc; a sample whose first covering
                         window ran in an earlier call starts from carry.  Call with j0 = 0, B, 2B, ... in order.
   seist_stream_emit   = probs (mean: one IEEE division by the number of covering windows; max as is) and carry_out.
   seist_stream_keep   = tail_out.
   The final probabilities are picked by seist_ragged_peaks and seist_ragged_runs, every row a stretch of f1 - f0. */
typedef struct SeistStreamStep {
  int64_t f0, r0, f1, r1;
  int64_t k0;          /* first regular window of the call */
  int64_t tail;        /* start of the tail window run by the call, -1: none */
  int64_t kr;          /* regular windows of the record (known at the close), -1 before */
  int32_t S, C, W, P;
  int32_t nk;          /* regular windows per station run by the call */
  int32_t norm_mode;   /* 0 none, 1 std, 2 max */
  int32_t stack_mode;  /* 0 mean, 1 max */
  int32_t pad_;
} SeistStreamStep;

uint64_t seist_sizeof_stream_step(void);
int seist_stream_window(const SeistStreamStep* step, const float* tail_raw, const float* chunk, int64_t j0, int32_t B, float* x,
                        void* stream);
int seist_stream_stack(const SeistStreamStep* step, const float* y, int64_t j0, int32_t B, const float* carry, float* acc,
                       void* stream);
int seist_stream_emit(const SeistStreamStep* step, const float* carry, const float* acc, float* probs, float* carry_out,
                      void* stream);
int seist_stream_keep(const SeistStreamStep* step, const float* tail_raw, const float* chunk, float* tail_out, void* stream);

/* ---- ragged streams: stations that advance at different rates (DESIGN §4.19) -----------------------------------------
   One call of a ragged stream is SeistStreamStep per station: every per-station count is a device int64 array of S
   entries (f0, r0, f1, r1, k0, nk, tail, kr as in SeistStreamStep), and four exclusive prefix arrays of S + 1 entries pack
   the call's data back to back:
     win_off   the call's windows, nk[s] + (tail[s] >= 0); call window j belongs to the last s with win_off[s] <= j and is
               that station's window j - win_off[s] (the tail one last).
     chunk_off the new samples: chunk holds station s as a (C, r1[s] - r0[s]) block at C * chunk_off[s].
     acc_off   the partial sums: acc holds station s as a (3, r1[s] - f0[s]) block at 3 * acc_off[s].
     out_off   the final probabilities: probs holds station s as a (3, f1[s] - f0[s]) block at 3 * out_off[s].
   tail_raw / tail_out (S, C, W) and carry / carry_out (S, 3, W) are per station as in SeistStreamStep.  The host-side
   totals n_win (= win_off[S]) and max_len (= max over s of r1[s] - f0[s]) size the grids; the arrays are never read back.
   Every device read of raw samples, partial sums and carries is range-checked against the station's own counts.
   seist_ragged_window = seist_stream_window for the call's windows j0 .. j0 + B - 1 (zero rows from n_win on).
   seist_ragged_stack  = seist_stream_stack of those windows' outputs, per station; s0 .. s1 are the stations of windows
                         j0 .. min(j0 + B, n_win) - 1 (the host knows win_off).  Call with j0 = 0, B, 2B, ... in order.
   seist_ragged_emit   = probs and carry_out; seist_ragged_keep = tail_out (the last min(W, r1[s]) raw samples).
   Picking a ragged stream: ext holds row s as a (C, L_s) block at C * ext_off[s], L_s = ext_off[s + 1] - ext_off[s]:
   the two samples before the stretch, the stretch of m_s samples and at the close one -inf sentinel.
   seist_ragged_ext    = ext from look (S, C, 2) and the stretches (probs packed at C * prob_off[s], (C, m_s)), every
                         sample past them -inf (the sentinel when L_s = m_s + 3), plus look_out (S, C, 2) = ext samples
                         m_s, m_s + 1 of each row.
   ext sample i of row s is global sample g0[s] + i.  lo, hi, lim, base, ishift, delta and g0 are per-row device int64
   arrays; max_span >= max(hi - lo + 1) and max_L = max L_s size the grids.
   seist_ragged_peaks  = the rising-edge candidates of ext[s, channel] at i in [max(lo, 1), min(hi, L_s - 2)] go behind the
                         ones still pending from the previous call's work `prev` (prev_capc, prev_L; null on the first
                         call), rebased by -delta[s]; candidates are held as int32 offsets from base[s] (candidate i:
                         i + ishift[s], ishift = g0 - base).  Clusters (gaps <= mpd) whose last candidate c has
                         c + mpd <= lim[s] are resolved as in seist_peaks_long; the rest stay pending.  counts (S,) int64:
                         picks; info (2S,) int64: pending count, global index of the first pending candidate (INT64_MAX
                         when none).  work: seist_stream_peaks_work_bytes(S, capc, max_L); capc >= max pending +
                         max_L / 2 + 1.  seist_ragged_peaks_fill writes the picks (global index = base[s] + offset) as
                         seist_peaks_long_fill does.
   seist_ragged_runs   = the runs of ext[s, channel] > threshold that end in this stretch: position p in
                         [max(lo, 1), min(hi, L_s - 1)] closes a run at p - 1 or opens one at p.  open_in (S,) int64: the
                         start of the run open before the stretch (-1: none); open_out: the same after it.  counts (S,)
                         int64; work: seist_runs_work_bytes(S, max_L).  seist_ragged_runs_fill writes the [on, off] pairs
                         (global) at pairs[offsets[s] ..]. */
typedef struct SeistRaggedStep {
  const int64_t *f0, *r0, *f1, *r1, *k0, *nk, *tail, *kr;   /* (S,) each */
  const int64_t *win_off, *chunk_off, *acc_off, *out_off;    /* (S + 1,) each */
  int64_t n_win;       /* win_off[S] */
  int64_t max_len;     /* max over s of r1[s] - f0[s] */
  int32_t S, C, W, P;
  int32_t norm_mode;   /* 0 none, 1 std, 2 max */
  int32_t stack_mode;  /* 0 mean, 1 max */
} SeistRaggedStep;

uint64_t seist_sizeof_ragged_step(void);
int seist_ragged_window(const SeistRaggedStep* step, const float* tail_raw, const float* chunk, int64_t j0, int32_t B, float* x,
                        void* stream);
int seist_ragged_stack(const SeistRaggedStep* step, const float* y, int64_t j0, int32_t B, int32_t s0, int32_t s1,
                       const float* carry, float* acc, void* stream);
int seist_ragged_emit(const SeistRaggedStep* step, const float* carry, const float* acc, float* probs, float* carry_out,
                      void* stream);
int seist_ragged_keep(const SeistRaggedStep* step, const float* tail_raw, const float* chunk, float* tail_out, void* stream);
int seist_ragged_ext(const float* look, const float* probs, const int64_t* prob_off, const int64_t* ext_off, int32_t S, int32_t C,
                     int64_t max_L, float* ext, float* look_out, void* stream);
int64_t seist_stream_peaks_work_bytes(int32_t S, int32_t capc, int64_t L);
int seist_ragged_peaks(const float* ext, const int64_t* ext_off, int32_t S, int32_t C, int32_t channel, int64_t max_L,
                       const int64_t* lo, const int64_t* hi, int64_t max_span, float mph, int32_t min_peak_dist,
                       const int64_t* lim, const int64_t* base, const int64_t* ishift, void* work, int32_t capc,
                       const void* prev, int32_t prev_capc, int64_t prev_L, const int64_t* delta, int32_t max_pend,
                       int64_t* counts, int64_t* info, void* stream);
int seist_ragged_peaks_fill(int32_t S, int64_t max_L, const void* work, int32_t capc, const int64_t* base, const int64_t* offsets,
                            int64_t* index, float* value, void* stream);
int seist_ragged_runs(const float* ext, const int64_t* ext_off, int32_t S, int32_t C, int32_t channel, int64_t max_L,
                      const int64_t* lo, const int64_t* hi, int64_t max_span, float threshold, const int64_t* open_in,
                      int64_t* open_out, void* work, int64_t work_bytes, int64_t* counts, void* stream);
int seist_ragged_runs_fill(const float* ext, const int64_t* ext_off, int32_t S, int32_t C, int32_t channel, int64_t max_L,
                           const int64_t* lo, const int64_t* hi, int64_t max_span, float threshold, const int64_t* g0,
                           const int64_t* open_in, int64_t* open_out, const void* work, int64_t work_bytes,
                           const int64_t* offsets, int64_t* pairs, void* stream);

/* ---- raw histories of characterised streams (DESIGN §4.18, §4.20) ----------------------------------------------------
   A packed history holds station s as a (C, len_s) block at C * off[s], len_s = off[s + 1] - off[s], whose first sample
   is the station's global sample h0[s]; off (S + 1,) and h0 (S,) are device int64 arrays, never read back to the host.
   seist_ragged_history       = the raw history of a characterised stream after a push: out row (s, c) = the samples
                                [h0_out[s], h0_out[s] + len_out_s) of the held row (held_off, h0_held) followed by the
                                station's block of the chunk packed as in SeistRaggedStep (chunk_off); each retained sample
                                is read and written once.  max_len >= every len_out_s sizes the grid (0 launches nothing);
                                reads outside a station's own held and chunk blocks or past a buffer's capacity (floats)
                                give 0.0f, writes past out_capacity are dropped.
                                out overlaps neither input; S * C <= 65535.
   seist_ragged_event_windows = seist_event_windows cutting from a packed history: station s the last one with
                                offsets[s] <= e (a bounded search), p = index[e] - h0[s] rebased on the device, row s read at
                                C * hist_off[s] with 0.0f outside [0, len_s) (and past hist_capacity).  Events >= M and
                                picks outside the station's history give zero rows.
   seist_gap_event_windows    = seist_ragged_event_windows for a stream with data gaps (DESIGN §4.23): event e belongs to
                                position q, the last with pos_off[q] <= e (a bounded search over n_pos + 1 offsets), whose
                                station pos_station[q] and segment [pos_on[q], pos_end[q]] (global, inclusive) come from the
                                position table (n_pos entries each); the pick p = index[e] is global.  Samples outside
                                [on, end] ∩ [h0_s, h0_s + len_s) read as 0.0f (and past hist_capacity), so each window is
                                that of seist_segment_event_windows on the station's whole record.  Events >= M, a station
                                outside [0, S) and picks outside that intersection give zero rows. */
int seist_ragged_history(const float* held, const int64_t* held_off, const int64_t* h0_held, int64_t held_capacity, const float* chunk,
                         const int64_t* chunk_off, int64_t chunk_capacity, const int64_t* h0_out, const int64_t* out_off, int32_t S,
                         int32_t C, int64_t max_len, float* out, int64_t out_capacity, void* stream);
int seist_ragged_event_windows(const float* hist, const int64_t* hist_off, const int64_t* h0, int64_t hist_capacity, int32_t S,
                               int32_t C, const int64_t* index, int64_t M, const int64_t* offsets, int64_t e0, int32_t B, int32_t W,
                               int32_t anchor, int32_t mode, float* const* x, int32_t n_dst, void* stream);
int seist_gap_event_windows(const float* hist, const int64_t* hist_off, const int64_t* h0, int64_t hist_capacity, int32_t S, int32_t C,
                            const int64_t* pos_station, const int64_t* pos_on, const int64_t* pos_end, const int64_t* pos_off,
                            int32_t n_pos, const int64_t* index, int64_t M, int64_t e0, int32_t B, int32_t W, int32_t anchor, int32_t mode,
                            float* const* x, int32_t n_dst, void* stream);

/* ---- whole records with data gaps (DESIGN §4.21) ----------------------------------------------------------------------
   Sample t of station s is a gap sample when any channel of record (S, C, T) is not finite; a segment is a maximal run of
   non-gap samples, inclusive [on, off].  The segment table: pairs (G, 2) int64 in station order then time order, seg_off
   (S + 1,) int64 (station s holds segments seg_off[s] .. seg_off[s + 1] - 1), station (G,) int64.  A segment of at least
   W samples is annotated: its windows are those of a record of off - on + 1 samples (K_g of them), packed back to back
   over all segments by win_off (G + 1,) int64 (K_g = 0 for a short segment).  Every table read is range-checked: a
   malformed table gives wrong output but no out-of-range access.
   seist_gap_segments          = per station, the number of segments (counts (S,) int64) and, in work
                                 (seist_runs_work_bytes(S, T)), per-block offsets for seist_gap_segments_fill, which
                                 writes pairs for offsets = the exclusive prefix of counts (rows >= capacity are dropped).
   seist_segment_window        = seist_window_batch over the packed windows j0 .. j0 + B - 1 (zero rows from n_win on):
                                 window j is window j - win_off[g] of segment g (the last with win_off[g] <= j), cut in
                                 place from the record at on_g + its start.
   seist_segment_stack         = seist_stack_batch of those windows' outputs into probs (S, 3, T) at each segment's
                                 samples; g0 .. g1 are the segments of windows j0 .. min(j0 + B, n_win) - 1.  Call with
                                 j0 = 0, B, 2B, ... in order.
   seist_segment_finish        = mode 0 (mean): divide every sample of an annotated segment by its number of covering
                                 windows in the segment; both modes: NaN at every sample outside an annotated segment.
   seist_segment_gather        = flat row r (a (3, m_r) block at 3 * prob_off[r], m_r = prob_off[r + 1] - prob_off[r]) =
                                 probs[station, :, on + i] of segment rows[r], i < m_r; writes past capacity are dropped.
   seist_segment_event_windows = seist_event_windows with the zero fill outside the pick's own segment: the segment of
                                 station s holding p when annotated[g] (one byte each) is set, else a zero row. */
int seist_gap_segments(const float* record, int32_t S, int32_t C, int64_t T, void* work, int64_t work_bytes, int64_t* counts,
                       void* stream);
int seist_gap_segments_fill(const float* record, int32_t S, int32_t C, int64_t T, const void* work, int64_t work_bytes,
                            const int64_t* offsets, int64_t* pairs, int64_t capacity, void* stream);
int seist_segment_window(const float* record, int32_t S, int32_t C, int64_t T, const int64_t* pairs, const int64_t* station,
                         const int64_t* win_off, int32_t G, int64_t n_win, int32_t W, int32_t P, int64_t j0, int32_t B, int32_t mode,
                         float* x, void* stream);
int seist_segment_stack(const float* y, int32_t S, int64_t T, const int64_t* pairs, const int64_t* station, const int64_t* win_off,
                        int32_t G, int64_t n_win, int32_t W, int32_t P, int64_t j0, int32_t B, int32_t g0, int32_t g1, int32_t mode,
                        float* probs, void* stream);
int seist_segment_finish(float* probs, int32_t S, int64_t T, const int64_t* pairs, const int64_t* seg_off, int32_t G, int32_t W,
                         int32_t P, int32_t mode, void* stream);
int seist_segment_gather(const float* probs, int32_t S, int64_t T, const int64_t* pairs, const int64_t* station, int32_t G,
                         const int64_t* rows, const int64_t* prob_off, int32_t n_rows, int64_t max_len, float* flat, int64_t capacity,
                         void* stream);
int seist_segment_event_windows(const float* record, int32_t S, int32_t C, int64_t T, const int64_t* pairs, const int64_t* seg_off,
                                const uint8_t* annotated, int32_t G, const int64_t* index, int64_t M, const int64_t* offsets, int64_t e0,
                                int32_t B, int32_t W, int32_t anchor, int32_t mode, float* const* x, int32_t n_dst, void* stream);

/* ---- streams with data gaps (DESIGN §4.22) ----------------------------------------------------------------------------
   A push of S stations is a packed chunk of chunk_capacity floats: station s's samples are a (C, n_s) block at
   C * chunk_off[s] (chunk_off (S + 1,) int64, n_s = chunk_off[s + 1] - chunk_off[s] <= max_n); a station whose block does
   not fit the chunk is read as empty.  Gap samples and segments are those of seist_gap_segments, in each block's own
   sample index.
   seist_gap_stream_scan = per station, the number of segments of its block (counts (S,) int64) and, in work
                           (seist_runs_work_bytes(S, max_n)), per-block offsets for seist_gap_stream_fill, which writes
                           pairs [on, off] for offsets = the exclusive prefix of counts (rows >= capacity are dropped).
   seist_gap_stream_pack = out row r (a (C, n_r) block at C * row_off[r], n_r = row_off[r + 1] - row_off[r]) = samples
                           row_start[r] .. row_start[r] + n_r - 1 of station row_station[r]'s block (0.0f outside it);
                           n = C * row_off[n_rows] elements, writes past out_capacity are dropped.
   seist_gap_stream_copy = for every row r, c < 3, t < m_r = m_off[r + 1] - m_off[r]:
                           dst[dst_base[r] + c * dst_ld[r] + t] = src[src_base[r] + c * src_ld[r] + t]; n = 3 * m_off[n_rows]
                           elements; reads past src_capacity give NaN, writes past dst_capacity are dropped. */
int seist_gap_stream_scan(const float* chunk, int64_t chunk_capacity, const int64_t* chunk_off, int32_t S, int32_t C, int64_t max_n,
                          void* work, int64_t work_bytes, int64_t* counts, void* stream);
int seist_gap_stream_fill(const float* chunk, int64_t chunk_capacity, const int64_t* chunk_off, int32_t S, int32_t C, int64_t max_n,
                          const void* work, int64_t work_bytes, const int64_t* offsets, int64_t* pairs, int64_t capacity, void* stream);
int seist_gap_stream_pack(const float* chunk, int64_t chunk_capacity, const int64_t* chunk_off, int32_t S, int32_t C,
                          const int64_t* row_station, const int64_t* row_start, const int64_t* row_off, int32_t n_rows, int64_t n,
                          float* out, int64_t out_capacity, void* stream);
int seist_gap_stream_copy(const float* src, int64_t src_capacity, const int64_t* m_off, const int64_t* src_base, const int64_t* src_ld,
                          const int64_t* dst_base, const int64_t* dst_ld, int32_t n_rows, int64_t n, float* dst, int64_t dst_capacity,
                          void* stream);

/* ---- polyphase resampling (DESIGN §4.24) -------------------------------------------------------------------------------
   scipy.signal.resample_poly(x, up, down, axis=-1) with its defaults (window ('kaiser', 5.0), zeros outside the record) for
   1 <= up, down <= 256 (the ratio reduced by the caller): output k of a row of T inputs, k < ceil(T * up / down), lies at input time k * down / up and is
   the fp32 fmaf chain over the in-record inputs i in ascending order of x[i] * h[k * down - i * up + hl], where the tap index
   lies in [0, 2 * hl] and hl = 10 * max(up, down).  Out-of-record inputs are skipped, not multiplied by zero, so an output is
   NaN exactly when a NaN input lies in its support.  taps: up phases of nt = 2 * hl / up + 1 floats each, phase phi holding
   h[phi + (nt_phi - 1 - t) * up] at taps[phi * nt + t] for t < nt_phi = (2 * hl - phi) / up + 1 (the order of ascending i).
   Every output of every call is computed by one device function, so a stream's outputs are bit-identical to the record's.
   seist_resample        = record (rows, T) -> out (rows, ceil(T * up / down)), one launch.
   seist_resample_stream = one call of S stations of C channels: desc is a device int64 array of N0, lo0, K0, lo1 (S each) then
                           chunk_off and out_off (S + 1 each).  Station s has received N0[s] inputs, holds inputs lo0 ..
                           N0 - 1 at held row (s, c) (held (S, C, H)), and has emitted outputs 0 .. K0 - 1; the push brings
                           n_s = chunk_off[s + 1] - chunk_off[s] inputs as a (C, n_s) block at C * chunk_off[s] of chunk.  The
                           call writes outputs K0 .. K0 + m_s - 1 (m_s = out_off[s + 1] - out_off[s]) as a (C, m_s) block at
                           C * out_off[s] of out, and inputs lo1 .. N0 + n_s - 1 to held_out row (s, c) (distinct from held).
                           Those outputs must have all their in-record inputs among lo0 .. N0 + n_s - 1; max_m >= every m_s sizes
                           the grid.  One launch; a malformed descriptor gives wrong output but no out-of-range access.
   Stations of different ratios share one launch through a filter table (DESIGN §4.24):
   seist_resample_table        = host only: fills table (F, 8) int32, one row per distinct reduced ratio i: up, down, hl, nt,
                                 tap_off, tile, identity, smem.  up == down gives the identity row (hl = nt = 0, no taps: the
                                 outputs are the inputs, copied bit for bit); otherwise the filter above.  tap_off is where
                                 the row's up * nt taps start in the concatenated taps (each padded to 4 floats), tile the
                                 outputs one CTA computes and smem the dynamic shared bytes such a CTA needs.
   seist_resample_multi        = whole records of S stations of C channels into out (S, C, T_max): desc is a device int64
                                 array of src (the device address of station s's (C, T_s) record), T_s, filt (the table row
                                 of station s) (S each), then cta_off (S + 1).  Row (s, c) holds ceil(T_s * up / down)
                                 outputs, then NaN up to T_max.  Station s owns CTAs cta_off[s] .. cta_off[s + 1] - 1, C * n_s
                                 of them: per channel ceil(T_out_s / tile) output tiles, then the rest fill the NaN tail in
                                 equal shares.  ctas = cta_off[S] sizes the grid and smem >= every smem of the rows used.
   seist_resample_multi_stream = seist_resample_stream with a filter per station: desc continues with filt (S) and cta_off
                                 (S + 1), station s owning C * max(1, ceil(m_s / tile)) CTAs; held is (S, C, H).
   One launch each, no host synchronisation; a malformed descriptor, table index or smem gives wrong output but no
   out-of-range access beyond the records desc points to. */
int seist_resample(const float* record, int32_t rows, int64_t T, const float* taps, int32_t up, int32_t down, float* out, void* stream);
int seist_resample_stream(const float* held, int64_t H, const float* chunk, int64_t chunk_capacity, const int64_t* desc, int32_t S,
                          int32_t C, int64_t max_m, const float* taps, int32_t up, int32_t down, float* out, int64_t out_capacity,
                          float* held_out, void* stream);
int seist_resample_table(int32_t F, const int32_t* up, const int32_t* down, int32_t* table);
int seist_resample_multi(const int64_t* desc, int32_t S, int32_t C, int64_t T_max, int64_t ctas, const int32_t* table, int32_t F,
                         int32_t smem, const float* taps, float* out, void* stream);
int seist_resample_multi_stream(const float* held, int64_t H, const float* chunk, int64_t chunk_capacity, const int64_t* desc,
                                int32_t S, int32_t C, int64_t ctas, const int32_t* table, int32_t F, int32_t smem, const float* taps,
                                float* out, int64_t out_capacity, float* held_out, void* stream);

/* *seed += 1 (device scalar), keeps dropout streams distinct across graph replays */
int seist_advance_seed(uint64_t* seed, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SEIST_B200_H_ */
