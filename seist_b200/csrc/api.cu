// C-ABI entry points and the plan executor (include/seist_b200.h).
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "common.cuh"

namespace seist {

static thread_local char g_err[512] = "";      // last error text of the calling thread
static std::atomic<uint64_t> g_launches{0};
static int g_sm_count = 0;

void set_error(const char* msg) {
  std::strncpy(g_err, msg, sizeof(g_err) - 1);
  g_err[sizeof(g_err) - 1] = 0;
}
void note_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
int check_launch(const char* what) {
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) {
    cudaGetLastError();
    std::snprintf(g_err, sizeof(g_err), "%s: %s", what, cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}

int launch_conv_fwd(const SeistOp& op, cudaStream_t s);
int launch_conv_bwd_data(const SeistOp& op, cudaStream_t s);
int launch_conv_bwd_w(const SeistOp& op, cudaStream_t s, int sm_count);
int launch_res_bwd(const SeistOp& op, cudaStream_t s);
int launch_att_fwd(const SeistOp& op, cudaStream_t s);
int launch_att_bwd_q(const SeistOp& op, cudaStream_t s);
int launch_att_bwd_kv(const SeistOp& op, cudaStream_t s);
int launch_headvec_fwd(const SeistOp& op, cudaStream_t s);
int launch_headvec_bwd(const SeistOp& op, cudaStream_t s);
int launch_bn_finalize(const SeistOp& op, bool fwd, cudaStream_t s);
bool pw_eligible(const SeistOp& op);
int launch_pw_fwd(const SeistOp& op, cudaStream_t s, int sm_count);
int launch_pw_bwd_data(const SeistOp& op, cudaStream_t s, int sm_count);
bool pw_bwd_data_staged_ok(const SeistOp& op);
int launch_pw_bwd_data_staged(const SeistOp& op, cudaStream_t s, int sm_count);
int launch_res_bwd4(const SeistOp& op, cudaStream_t s, int sm_count);
bool bww_eligible(const SeistOp& op);
int launch_bww_any(const SeistOp& op, cudaStream_t s, int sm_count);
bool convk_eligible(const SeistOp& op);
bool bwwk_eligible(const SeistOp& op);
bool convk_bwd_data_eligible(const SeistOp& op);
int launch_bwwk(const SeistOp& op, cudaStream_t s, int sm_count);
int launch_convk_fwd(const SeistOp& op, cudaStream_t s);
int launch_convk_bwd_data(const SeistOp& op, cudaStream_t s);
int launch_bn_prepare(const SeistOp& op, bool fwd, cudaStream_t s);
int launch_stem_compose(const SeistOp& op, bool fwd, cudaStream_t s);
bool tcconv_eligible(const SeistOp& op, int mode);
int launch_tcconv(const SeistOp& op, int mode, cudaStream_t s, int sm_count);
int tcconv_error_flag();

// Tensor-core convolution engine (tcconv.cu: wgmma + TMA, 3 x TF32) for stride-1 forward / data-gradient convs.  Measured
// op by op on H100 at the bench configuration (seist_m_dpk, B = 512, engine forced vs SIMT kernels): it wins on the
// up-sampled head convs with >= 32 input channels, the k-tap convs of encoder stages 1-3 (forward at L <= 512 with >= 16
// reduction channels, data gradient at L <= 256 with >= 32) and the forward 1x1 convs with >= 64 reduction channels at
// L <= 256; everywhere else (stem, stage 0, the long head layers, most 1x1 data gradients) the SIMT kernels are faster.
// SEIST_TCC: unset = that rule, "1" = every eligible op (tests), "0" = never.
static int tcc_mode() {
  static int v = -1;
  if (v < 0) { const char* e = std::getenv("SEIST_TCC"); v = !e ? 2 : (e[0] == '0' ? 0 : (e[0] == '1' ? 1 : 2)); }
  return v;
}
static bool tcc_auto(const SeistOp& op, int mode) {
  const int Kd = mode == 0 ? op.Cin : op.Cout;
  if (op.up_src_L > 0) return mode == 0 && Kd >= 32;
  if (op.k > 1) return mode == 0 ? (op.L_out <= 512 && Kd >= 16) : (op.L_out <= 256 && Kd >= 32);
  return mode == 0 && Kd >= 64 && op.L_out <= 256;
}
static bool use_tcc(const SeistOp& op, int mode) {
  const int m = tcc_mode();
  if (m == 0 || !tcconv_eligible(op, mode)) return false;
  return m == 1 || tcc_auto(op, mode);
}

static int sm_count() {
  if (g_sm_count == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&g_sm_count, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || g_sm_count <= 0)
      g_sm_count = 132;
  }
  return g_sm_count;
}

static int validate_conv(const SeistOp& op) {
  if (op.groups <= 0 || op.Cin % op.groups || op.Cout % op.groups) { set_error("conv: channels not divisible by groups"); return -2; }
  if (op.k < 1 || op.stride < 1 || op.N < 1 || op.L_out < 1) { set_error("conv: bad geometry"); return -2; }
  if (op.n_in < 1 || op.n_in > SEIST_MAX_IN) { set_error("conv: bad n_in"); return -2; }
  if ((op.pool > 1 || op.up_src_L > 0) && op.n_in != 1) { set_error("conv: pool/upsample need a single input view"); return -2; }
  if (op.pool > 1 && (op.k != 1 || op.up_src_L > 0)) { set_error("conv: pool only with k=1"); return -2; }
  if (op.N > 65535) { set_error("conv: batch > 65535 per launch"); return -2; }
  return 0;
}

// which kernel family serves an op (also reported to the bench: `seist_op_family`)
enum Family {
  F_NONE = 0, F_TCCONV_FWD, F_TCCONV_BWD_DATA, F_PW_FWD, F_CONVK_FWD, F_CONV_FWD, F_PW_BWD_DATA, F_PW_BWD_DATA_STAGED, F_CONVK_BWD_DATA,
  F_CONV_BWD_DATA, F_BWWK, F_BWW, F_CONV_BWD_W, F_RES_BWD, F_RES_BWD4, F_ATT_FWD, F_ATT_BWD_Q, F_ATT_BWD_KV, F_HEADVEC_FWD,
  F_HEADVEC_BWD, F_BN_FINALIZE_FWD, F_BN_FINALIZE_BWD, F_BN_PREPARE_FWD, F_BN_PREPARE_BWD, F_STEM_COMPOSE_FWD, F_STEM_COMPOSE_BWD,
  F_ZERO
};
static const char* kFamilyName[] = {
  "none", "tcconv_fwd(wgmma+TMA)", "tcconv_bwd_data(wgmma+TMA)", "pw_fwd(simt)", "convk_fwd(simt)",
  "conv_fwd(simt)", "pw_bwd_data(simt)", "pw_bwd_data_staged(simt)", "convk_bwd_data(simt)", "conv_bwd_data(simt)", "bwwk(simt)", "bww(simt)",
  "conv_bwd_w(simt)", "res_bwd", "res_bwd4", "att_fwd", "att_bwd_q", "att_bwd_kv", "headvec_fwd", "headvec_bwd", "bn_finalize_fwd",
  "bn_finalize_bwd", "bn_prepare_fwd", "bn_prepare_bwd", "stem_compose_fwd", "stem_compose_bwd", "zero"
};

static Family choose(const SeistOp& op) {
  switch (op.kind) {
    case SEIST_OP_CONV_FWD:
      if (use_tcc(op, 0)) return F_TCCONV_FWD;
      if (pw_eligible(op)) return F_PW_FWD;
      return convk_eligible(op) ? F_CONVK_FWD : F_CONV_FWD;
    case SEIST_OP_CONV_BWD_DATA:
      if (use_tcc(op, 1)) return F_TCCONV_BWD_DATA;
      if (pw_bwd_data_staged_ok(op)) return F_PW_BWD_DATA_STAGED;
      if (pw_eligible(op)) return F_PW_BWD_DATA;
      return convk_bwd_data_eligible(op) ? F_CONVK_BWD_DATA : F_CONV_BWD_DATA;
    case SEIST_OP_CONV_BWD_W:
      if (bwwk_eligible(op)) return F_BWWK;
      return bww_eligible(op) ? F_BWW : F_CONV_BWD_W;
    case SEIST_OP_RES_BWD: return (op.L_out & 3) ? F_RES_BWD : F_RES_BWD4;
    case SEIST_OP_ATT_FWD: return F_ATT_FWD;
    case SEIST_OP_ATT_BWD_Q: return F_ATT_BWD_Q;
    case SEIST_OP_ATT_BWD_KV: return F_ATT_BWD_KV;
    case SEIST_OP_HEADVEC_FWD: return F_HEADVEC_FWD;
    case SEIST_OP_HEADVEC_BWD: return F_HEADVEC_BWD;
    case SEIST_OP_BN_FINALIZE_FWD: return F_BN_FINALIZE_FWD;
    case SEIST_OP_BN_FINALIZE_BWD: return F_BN_FINALIZE_BWD;
    case SEIST_OP_BN_PREPARE_FWD: return F_BN_PREPARE_FWD;
    case SEIST_OP_BN_PREPARE_BWD: return F_BN_PREPARE_BWD;
    case SEIST_OP_STEM_COMPOSE_FWD: return F_STEM_COMPOSE_FWD;
    case SEIST_OP_STEM_COMPOSE_BWD: return F_STEM_COMPOSE_BWD;
    case SEIST_OP_ZERO: return F_ZERO;
    default: return F_NONE;
  }
}

static int run_one(const SeistOp& op, cudaStream_t s) {
  if (op.kind == SEIST_OP_CONV_FWD || op.kind == SEIST_OP_CONV_BWD_DATA || op.kind == SEIST_OP_CONV_BWD_W) {
    int v = validate_conv(op);
    if (v) return v;
  }
  switch (choose(op)) {
    case F_TCCONV_FWD: return launch_tcconv(op, 0, s, sm_count());
    case F_TCCONV_BWD_DATA: return launch_tcconv(op, 1, s, sm_count());
    case F_PW_FWD: return launch_pw_fwd(op, s, sm_count());
    case F_CONVK_FWD: return launch_convk_fwd(op, s);
    case F_CONV_FWD: return launch_conv_fwd(op, s);
    case F_PW_BWD_DATA: return launch_pw_bwd_data(op, s, sm_count());
    case F_PW_BWD_DATA_STAGED: return launch_pw_bwd_data_staged(op, s, sm_count());
    case F_CONVK_BWD_DATA: return launch_convk_bwd_data(op, s);
    case F_CONV_BWD_DATA: return launch_conv_bwd_data(op, s);
    case F_BWWK: return launch_bwwk(op, s, sm_count());
    case F_BWW: return launch_bww_any(op, s, sm_count());
    case F_CONV_BWD_W: return launch_conv_bwd_w(op, s, sm_count());
    case F_RES_BWD: return launch_res_bwd(op, s);
    case F_RES_BWD4: return launch_res_bwd4(op, s, sm_count());
    case F_ATT_FWD: return launch_att_fwd(op, s);
    case F_ATT_BWD_Q: return launch_att_bwd_q(op, s);
    case F_ATT_BWD_KV: return launch_att_bwd_kv(op, s);
    case F_HEADVEC_FWD: return launch_headvec_fwd(op, s);
    case F_HEADVEC_BWD: return launch_headvec_bwd(op, s);
    case F_BN_FINALIZE_FWD: return launch_bn_finalize(op, true, s);
    case F_BN_FINALIZE_BWD: return launch_bn_finalize(op, false, s);
    case F_BN_PREPARE_FWD: return launch_bn_prepare(op, true, s);
    case F_BN_PREPARE_BWD: return launch_bn_prepare(op, false, s);
    case F_STEM_COMPOSE_FWD: return launch_stem_compose(op, true, s);
    case F_STEM_COMPOSE_BWD: return launch_stem_compose(op, false, s);
    case F_ZERO: {
      cudaError_t e = cudaMemsetAsync(op.out.x, 0, op.zero_bytes, s);
      if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); return (int)e; }
      return 0;
    }
    default: set_error("unknown op kind"); return -1;
  }
}

}  // namespace seist

extern "C" {

int seist_plan_run(const SeistOp* ops, int32_t n, void* stream);
const char* seist_last_error(void);

int seist_abi_version(void) { return SEIST_ABI_VERSION; }
uint64_t seist_sizeof_op(void) { return sizeof(SeistOp); }
uint64_t seist_sizeof_bn(void) { return sizeof(SeistBN); }
const char* seist_last_error(void) { return seist::g_err; }
uint64_t seist_launch_count(void) { return seist::g_launches.load(); }
const char* seist_op_family(const SeistOp* op) { return op ? seist::kFamilyName[seist::choose(*op)] : "none"; }
int seist_tc_error_flag(void) { return seist::tcconv_error_flag(); }

// lane and fork/join events of seist_plan_run_lanes, one pool per device (events belong to the device that was current
// at creation)
static std::vector<cudaEvent_t> g_events[64];
static cudaEvent_t event_at(size_t i) {
  int dev = 0;
  cudaGetDevice(&dev);
  std::vector<cudaEvent_t>& pool = g_events[dev & 63];
  while (pool.size() <= i) {
    cudaEvent_t e = nullptr;
    if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return nullptr;
    pool.push_back(e);
  }
  return pool[i];
}
static int fork_join(cudaStream_t from, cudaStream_t to, size_t& ev) {
  cudaEvent_t e = event_at(ev++);
  if (e == nullptr) { seist::set_error("plan_run_lanes: cudaEventCreate failed"); return (int)cudaErrorMemoryAllocation; }
  cudaError_t r = cudaEventRecord(e, from);
  if (r == cudaSuccess) r = cudaStreamWaitEvent(to, e, 0);
  if (r != cudaSuccess) { seist::set_error(cudaGetErrorString(r)); return (int)r; }
  return 0;
}

int seist_plan_run_lanes(const SeistOp* ops, int32_t n, void* const* streams, int32_t n_streams) {
  if (ops == nullptr || n < 0 || streams == nullptr || n_streams < 1 || n_streams > 8) { seist::set_error("plan_run_lanes: bad arguments"); return -1; }
  if (n_streams == 1) return seist_plan_run(ops, n, streams[0]);
  cudaStream_t s0 = (cudaStream_t)streams[0];
  // events 0 .. n-1: per-op records (ids assigned by the scheduler), n .. n+8: fork / join
  size_t ev = (size_t)n;
  for (int l = 1; l < n_streams; ++l) {
    size_t e = ev;
    const int fr = fork_join(s0, (cudaStream_t)streams[l], e);      // same fork event slot re-recorded per lane: fine
    if (fr) return fr;
  }
  int rc = 0;
  for (int i = 0; i < n && rc == 0; ++i) {
    const SeistOp& op = ops[i];
    const int lane = op.lane < 0 ? 0 : (op.lane >= n_streams ? n_streams - 1 : op.lane);
    cudaStream_t s = (cudaStream_t)streams[lane];
    for (int w = 0; w < op.n_wait && w < 4 && rc == 0; ++w) {
      if (op.wait_ev[w] < 0 || op.wait_ev[w] >= n) { seist::set_error("plan_run_lanes: bad event id"); rc = -1; break; }
      cudaEvent_t e = event_at((size_t)op.wait_ev[w]);
      cudaError_t r = e ? cudaStreamWaitEvent(s, e, 0) : cudaErrorMemoryAllocation;
      if (r != cudaSuccess) { seist::set_error(cudaGetErrorString(r)); rc = (int)r; }
    }
    if (rc) break;
    rc = seist::run_one(op, s);
    if (rc != 0) {
      char buf[600];
      std::snprintf(buf, sizeof(buf), "op %d (kind %d): %s", i, op.kind, seist_last_error());
      seist::set_error(buf);
      break;
    }
    if (op.rec_event >= 0) {
      cudaEvent_t e = op.rec_event < n ? event_at((size_t)op.rec_event) : nullptr;
      cudaError_t r = e ? cudaEventRecord(e, s) : cudaErrorMemoryAllocation;
      if (r != cudaSuccess) { seist::set_error(cudaGetErrorString(r)); rc = (int)r; }
    }
  }
  for (int l = 1; l < n_streams; ++l) {          // join (also on errors: never leave a captured fork dangling)
    size_t e = (size_t)n + 1 + (size_t)l;
    const int jr = fork_join((cudaStream_t)streams[l], s0, e);
    if (jr && !rc) rc = jr;
  }
  return rc;
}

int seist_plan_run(const SeistOp* ops, int32_t n, void* stream) {
  if (ops == nullptr || n < 0) { seist::set_error("plan_run: bad arguments"); return -1; }
  cudaStream_t s = (cudaStream_t)stream;
  for (int i = 0; i < n; ++i) {
    int rc = seist::run_one(ops[i], s);
    if (rc != 0) {
      char buf[600];
      std::snprintf(buf, sizeof(buf), "op %d (kind %d): %s", i, ops[i].kind, seist::g_err);
      seist::set_error(buf);
      return rc;
    }
  }
  return 0;
}

}  // extern "C"
