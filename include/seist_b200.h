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

#define SEIST_ABI_VERSION 11
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

/* *seed += 1 (device scalar), keeps dropout streams distinct across graph replays */
int seist_advance_seed(uint64_t* seed, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SEIST_B200_H_ */
