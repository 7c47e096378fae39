// Convolution forward / data-gradient on the Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a.
//
//   forward        out[co][l] = sum_{ci,t} W[co][ci][t] * f(in[ci])[l*1 + t - pad]        (nn.Conv1d, models/seist.py:86..546)
//   data gradient  dIn[ci][p] = sum_{co,t} W[co][ci][t] * gacc[co][p + pad - t]            (its autograd transpose)
//
// Both are the same GEMM per 128-sample tile:  D[M = 128 samples][N = result channels] += A_t[M][K] * B_t[N][K]^T summed
// over the k taps t, where A_t is the SAME shared-memory panel read at a row offset of t samples:
//
//   panel layout (K-major, no swizzle):  [channel/4][row][channel%4]  (16 bytes = 4 reduction channels of one sample)
//   a core matrix (8 rows x 16 B) of channel-quad q starting at ANY row r0 is the contiguous 128 bytes at q*pitch + r0*16,
//   so the descriptor of tap t is just  start += 16*t  (LBO = pitch between channel quads, SBO = 128 between 8-row groups).
//   No im2col copy, no weight expansion: k * ceil(K/8) MMA steps per tile and precision pass.
//
// Warp roles (one persistent CTA per SM, 544 threads):
//   warp 16      TMA producer: cp.async.bulk.tensor boxes {rows, 8 channels} of the raw fp32 operand tensors -> raw ring
//                (zero fill outside the tensor = the conv's zero padding of the raw rows; mbarrier complete_tx)
//   warps 8..15  transform: raw ring -> BN-apply / GELU (forward) or BN-backward / dropout / sigmoid' (data gradient)
//                -> exact hi + lo TF32 split -> panel ring (generic stores + fence.proxy.async)
//   warps 0..7   two consumer warpgroups: warpgroup h issues one wgmma.m64nNk8 .tf32 per k-step and pass (N = result
//                channels padded to 32 / 64 / 128, a template parameter) for rows 64h .. 64h+63 of the tile,
//                3 passes (hi*hi + lo*hi + hi*lo ~ fp32 products), accumulators in registers; then both park them in a
//                shared staging tile [channel][sample] and run the epilogue (lane = sample): bias / dropout / residual views
//                / BatchNorm statistics (forward) or GELU' / BN-backward sums / accumulate (data gradient), coalesced
//                128-byte stores.  The producer and transform warps stage the next tile meanwhile.
#include <cuda.h>
#include <cstdlib>
#include <cstring>
#include "common.cuh"

namespace seist {

constexpr int TCC_EPI_WARPS = 8;      // two consumer warpgroups (MMA + epilogue)
constexpr int TCC_XF_WARPS = 8;
constexpr int TCC_NT = 32 * (TCC_EPI_WARPS + TCC_XF_WARPS + 1);
constexpr int TCC_M = 128;
constexpr int TCC_MAX_STAGES = 8;
constexpr int TCC_NMAX = 128;         // result channels: 64 accumulator registers per consumer thread
constexpr int TCC_ACC_PITCH = TCC_M + 4;  // staging tile row pitch (floats): conflict-free fragment stores

struct TccGeom {
  int mode;             // 0 forward, 1 data gradient
  int Kd, Nd;           // reduction channels, result channels
  int k, padl;          // taps; left pad of the conv in the operand-row coordinate (forward pad_left, backward k-1-pad_left)
  int padA, toff;       // TMA boxes must start 16-byte aligned: panel row 0 = sample l0 - padA, padA = padl rounded up to 4,
                        // tap t reads panel rows m + t + toff (toff = padA - padl)
  int src_len, dst_len; // length of the operand rows / of the result rows
  int KC, nchunks;      // reduction channels per chunk (multiple of 8), chunks
  int R, Rbox, Rp;      // panel rows needed (128+k-1), TMA box rows (R rounded to 4), row pitch of the panel (R rounded to 32)
  int N_pad;            // MMA N (multiple of 16)
  int raw_stages, a_stages, b_resident;
  int n_raw;            // raw tensors per stage (forward 1; backward: dxd / du / x as present)
  int raw_tensor_bytes; // KC * Rbox * 4
  int a_part;           // bytes of one precision part of a panel stage: (KC/4) * Rp * 16
  int b_part;           // bytes of one precision part of one chunk's weights: k * (KC/4) * N_pad * 16
  int a_stage;          // bytes of one panel stage: 2 * a_part (+ 2 * b_part when the weights are streamed)
  int has_dxd, has_bn, need_x;
  int up, up_S;         // forward only: the operand is the x2 linear up-sampling (F.interpolate, align_corners=False,
                        // models/seist.py:566) of a source of up_S samples; the raw ring then holds SOURCE rows
  // shared-memory carve-up (byte offsets from the 128-aligned base)
  int off_raw, off_a, off_b, off_tab_k, off_tab_n, off_red, off_acc, off_bar, smem_bytes;
};

struct TccMaps {
  CUtensorMap m[3];     // forward: one per input view; backward: dxd, du, x of the output tensor
};

// per reduction channel (transform warps)
struct TccK {
  float a, b, c;        // forward: sc, sh, act ; backward: A, Bx, Cc
  int view;             // forward: input view (tensor map) index
};
// per result channel of the data gradient (epilogue)
struct TccTgt {
  const float* x;
  float* g;
  long long nstride;
  float sc, sh, mu, istd;
  int act, bn, bnc, accum;
};

__device__ int g_tcc_err_dev = 0;

__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// wgmma shared-memory descriptor: start, LBO (K direction), SBO (M / N direction) in 16-byte units; no swizzle
__device__ __forceinline__ uint64_t tcc_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFFu);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;
}
// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, tf32 operands, fp32 accumulators in the m64nNk8 fragment layout (N / 2 per thread)
template <int N>
__device__ __forceinline__ void tcc_mma(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accum);
template <>
__device__ __forceinline__ void tcc_mma<32>(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(accum));
}
template <>
__device__ __forceinline__ void tcc_mma<64>(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accum));
}
template <>
__device__ __forceinline__ void tcc_mma<128>(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accum));
}
template <int R>
__device__ __forceinline__ void tcc_keep(float (&d)[R]) {      // accumulator registers are not touched across this point
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void tcc_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void tcc_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tcc_tma3(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(dst),
      "l"((uint64_t)map), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
      : "memory");
}
// bounded wait: never hangs the GPU; a timeout raises the CTA's abort flag (every role then leaves its loop)
__device__ __forceinline__ bool tcc_wait(uint32_t bar, uint32_t parity, volatile int* abort_s) {
  uint32_t done = 0;
  for (int it = 0; it < (1 << 18); ++it) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\tselp.b32 %0, 1, 0, p;\n\t}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity), "r"(20000u)      // suspend-time hint (ns): sleep in hardware, wake on completion
        : "memory");
    if (done) return true;
    if ((it & 15) == 15 && *abort_s) return false;
  }
  *abort_s = 1;
  return false;
}
__device__ __forceinline__ void tcc_split(float x, float& hi, float& lo) {
  hi = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
  lo = x - hi;
}
__device__ __forceinline__ float tcc_gelu(float x) { return gelu_f(x); }          // common.cuh: fast erf (A&S 7.1.26)
__device__ __forceinline__ float tcc_gelu_grad(float x) { return gelu_grad_f(x); }

// 16 values per lane -> every lane gets the warp-wide sum of value tcc_red_index(lane) (17 shuffles instead of 80)
__device__ __forceinline__ float tcc_reduce16(float (&v)[16], int lane) {
#pragma unroll
  for (int half = 8, off = 16; half >= 1; half >>= 1, off >>= 1) {
    const bool up = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (i < half) {
        const float send = up ? v[i] : v[i + half];
        const float keep = up ? v[i + half] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
      }
    }
  }
  return v[0] + __shfl_xor_sync(0xffffffffu, v[0], 1);
}
__device__ __forceinline__ int tcc_red_index(int lane) {
  return ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
}

// 16 staged accumulator columns of one sample row
#define TCC_LD16(rr, col0)                                                                                               \
  _Pragma("unroll") for (int c_ = 0; c_ < 16; ++c_) rr[c_] = __float_as_uint(acc_s[((col0) + c_) * TCC_ACC_PITCH + srow]);

// first source row staged for a tile whose panel row 0 is up-sampled position p0 (a multiple of 4): the rows needed start at
// floor((p0 - 1) / 2); TMA boxes must start 16-byte aligned -> rounded down to a multiple of 4
__device__ __forceinline__ int tcc_up_src0(int p0) { return ((p0 >> 1) - 1) & ~3; }

// dense weight element of the panel B[t][n][c] (grouped convolutions are expanded with zero blocks)
__device__ __forceinline__ float tcc_wval(const SeistOp& op, int mode, int t, int n, int c) {
  const int co = mode == 0 ? n : c, ci = mode == 0 ? c : n;
  const int tt = mode == 0 ? t : op.k - 1 - t;
  if (co >= op.Cout || ci >= op.Cin) return 0.f;
  const int cin_g = op.Cin / op.groups, cout_g = op.Cout / op.groups;
  const int g = co / cout_g;
  if (ci / cin_g != g) return 0.f;
  return __ldg(op.W + ((size_t)co * cin_g + (ci - g * cin_g)) * op.k + tt);
}

// F_GELU: some input view applies GELU (forward transform / backward epilogue); F_ELEM: element dropout
// NB: MMA width (result channels padded to 32, 64 or 128)
template <int MODE, bool F_GELU, bool F_ELEM, int NB>
__global__ void __launch_bounds__(TCC_NT, 1) tcconv_kernel(const __grid_constant__ SeistOp op, const __grid_constant__ TccGeom g,
                                                           const __grid_constant__ TccMaps maps) {
  extern __shared__ __align__(16) unsigned char tcc_raw[];
  unsigned char* base = tcc_raw + ((128u - (s32(tcc_raw) & 127u)) & 127u);
  unsigned char* raw_s = base + g.off_raw;
  unsigned char* a_s = base + g.off_a;
  unsigned char* b_s = base + g.off_b;
  TccK* tk_s = reinterpret_cast<TccK*>(base + g.off_tab_k);                 // [Kd_pad]
  float* red_s = reinterpret_cast<float*>(base + g.off_red);               // [8 epilogue warps][2*Nd]
  uint64_t* bars = reinterpret_cast<uint64_t*>(base + g.off_bar);
  uint64_t* raw_full = bars;
  uint64_t* raw_empty = raw_full + TCC_MAX_STAGES;
  uint64_t* a_full = raw_empty + TCC_MAX_STAGES;
  uint64_t* a_empty = a_full + TCC_MAX_STAGES;
  volatile int* abort_s = reinterpret_cast<volatile int*>(a_empty + TCC_MAX_STAGES);
  float* acc_s = reinterpret_cast<float*>(base + g.off_acc);                // accumulator staging [N_pad][TCC_ACC_PITCH]

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);     // provably warp-uniform: the role branches hold wgmma
  const int Kd = g.Kd, Nd = g.Nd;
  const int Kd_pad = g.nchunks * g.KC;
  const int tiles_per_n = (g.dst_len + TCC_M - 1) / TCC_M;
  const int total = op.N * tiles_per_n;
  const bool has_bn_out = (op.out.bn >= 0 && op.out.g != nullptr);

  // ---- tables ----------------------------------------------------------------------------------------------------
  for (int c = tid; c < Kd_pad; c += TCC_NT) {
    TccK e;
    e.a = 0.f; e.b = 0.f; e.c = 0.f; e.view = 0;
    if (c < Kd) {
      if (MODE == 0) {
        int cv;
        const int vi = resolve_view(op, c, cv);
        view_coef(op, op.in[vi], cv, e.a, e.b);
        e.c = (float)op.in[vi].act;
        e.view = vi;
      } else {
        const OutGradCoef kc = out_grad_coef(op, c);
        e.a = kc.A; e.b = kc.Bx; e.c = kc.Cc;
      }
    }
    tk_s[c] = e;
  }
  if (MODE == 0) {
    float* ep_s = reinterpret_cast<float*>(base + g.off_tab_n);            // bias, a_sc, a_sh, b_sc, b_sh [5][Nd]
    for (int co = tid; co < Nd; co += TCC_NT) {
      float b = 0.f, asc = 1.f, ash = 0.f, bsc = 1.f, bsh = 0.f;
      if (op.bias) b = op.bias[co];
      if (op.res_a.C > 0) view_coef(op, op.res_a, co, asc, ash);
      if (op.res_b.C > 0) view_coef(op, op.res_b, co, bsc, bsh);
      ep_s[co] = b;
      ep_s[Nd + co] = asc;
      ep_s[2 * Nd + co] = ash;
      ep_s[3 * Nd + co] = bsc;
      ep_s[4 * Nd + co] = bsh;
    }
  } else {
    TccTgt* tg_s = reinterpret_cast<TccTgt*>(base + g.off_tab_n);          // [Nd]
    for (int ci = tid; ci < Nd; ci += TCC_NT) {
      int cv;
      const int vi = resolve_view(op, ci, cv);
      const SeistView& v = op.in[vi];
      TccTgt e;
      e.x = v.x + (size_t)(v.c0 + cv) * v.L;
      e.g = v.g ? v.g + (size_t)(v.c0 + cv) * v.L : nullptr;
      e.nstride = (long long)v.Ct * v.L;
      view_coef(op, v, cv, e.sc, e.sh);
      e.mu = 0.f; e.istd = 0.f;
      if (v.bn >= 0) view_khat(op, v, cv, e.mu, e.istd);
      e.act = v.act; e.bn = v.bn; e.bnc = v.bn_c0 + cv; e.accum = v.accum;
      tg_s[ci] = e;
    }
  }
  for (int i = tid; i < TCC_EPI_WARPS * 2 * Nd; i += TCC_NT) red_s[i] = 0.f;

  // weights -> panel B[chunk][t][c/4][n][c%4] (hi, lo).  Resident: every chunk once; streamed: per chunk by the transform warps.
  const int colpitchB = g.N_pad * 16;
  auto stage_b = [&](int chunk, unsigned char* b_hi, unsigned char* b_lo, int t0, int nthreads) {
    const int nq = g.KC >> 2;
    const int items = g.k * nq * g.N_pad;
    for (int idx = t0; idx < items; idx += nthreads) {
      const int n = idx % g.N_pad;
      const int rest = idx / g.N_pad;
      const int q = rest % nq, t = rest / nq;
      float4 hi, lo;
      float w[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = chunk * g.KC + 4 * q + j;
        w[j] = (n < Nd && c < Kd) ? tcc_wval(op, MODE, t, n, c) : 0.f;
      }
      tcc_split(w[0], hi.x, lo.x);
      tcc_split(w[1], hi.y, lo.y);
      tcc_split(w[2], hi.z, lo.z);
      tcc_split(w[3], hi.w, lo.w);
      const int off = (t * nq + q) * colpitchB + n * 16;
      *reinterpret_cast<float4*>(b_hi + off) = hi;
      *reinterpret_cast<float4*>(b_lo + off) = lo;
    }
  };
  if (g.b_resident)
    for (int ch = 0; ch < g.nchunks; ++ch) stage_b(ch, b_s + (size_t)ch * 2 * g.b_part, b_s + (size_t)ch * 2 * g.b_part + g.b_part, tid, TCC_NT);

  if (tid == 32) {
    for (int i = 0; i < TCC_MAX_STAGES; ++i) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(&raw_full[i])), "r"(1) : "memory");
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(&raw_empty[i])), "r"(TCC_XF_WARPS) : "memory");
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(&a_full[i])), "r"(TCC_XF_WARPS) : "memory");
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(&a_empty[i])), "r"(TCC_EPI_WARPS) : "memory");
    }
    *abort_s = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // resident weights: generic writes -> async proxy
  __syncthreads();
  const uint64_t seed = load_seed(op.step_seed);

  if (warp == TCC_EPI_WARPS + TCC_XF_WARPS) {
    // =========================== TMA producer ===========================
    if (lane == 0) {
      int rs = 0;
      uint32_t rph = 0;
      const uint32_t stage_tx = (uint32_t)(g.n_raw * g.raw_tensor_bytes);
      const int nbox = g.KC >> 3;
      for (int tile = blockIdx.x; tile < total && !*abort_s; tile += gridDim.x) {
        const int n = tile / tiles_per_n;
        const int p0 = (tile - n * tiles_per_n) * TCC_M - g.padA;
        for (int ch = 0; ch < g.nchunks; ++ch) {
          if (!tcc_wait(s32(&raw_empty[rs]), rph ^ 1, abort_s)) break;
          const uint32_t bar = s32(&raw_full[rs]);
          tcc_expect_tx(bar, stage_tx);
          const uint32_t dst0 = s32(raw_s + (size_t)rs * g.n_raw * g.raw_tensor_bytes);
          for (int b = 0; b < nbox; ++b) {
            const int c = ch * g.KC + 8 * b;         // first reduction channel of the box
            const uint32_t boxoff = (uint32_t)(8 * b * g.Rbox * 4);
            if (MODE == 0) {
              int cv = 0, vi = 0;
              if (c < Kd) vi = resolve_view(op, c, cv);
              else cv = 1 << 20;                    // padded channels: fully out of bounds -> zero fill
              tcc_tma3(dst0 + boxoff, &maps.m[vi], g.up ? tcc_up_src0(p0) : p0, op.in[vi].c0 + cv, n, bar);
            } else {
              const int cc = c < Kd ? op.out.c0 + c : (1 << 20);
              int slot = 0;
              if (g.has_dxd) { tcc_tma3(dst0 + slot * g.raw_tensor_bytes + boxoff, &maps.m[0], p0, cc, n, bar); ++slot; }
              if (g.has_bn) { tcc_tma3(dst0 + slot * g.raw_tensor_bytes + boxoff, &maps.m[1], p0, cc, n, bar); ++slot; }
              if (g.need_x) { tcc_tma3(dst0 + slot * g.raw_tensor_bytes + boxoff, &maps.m[2], p0, cc, n, bar); ++slot; }
            }
          }
          if (++rs == g.raw_stages) { rs = 0; rph ^= 1; }
        }
      }
    }
  } else if (warp >= TCC_EPI_WARPS) {
    // =========================== transform warps ===========================
    // warp -> one channel quad q (its 4 coefficient rows stay in registers for the whole chunk) and every
    // (8 / nq)-th 32-row block of the panel; lane = panel row
    const int xw = warp - TCC_EPI_WARPS;
    int rs = 0, as = 0;
    uint32_t rph = 0, aph = 0;
    const int nq = g.KC >> 2, nrb = g.Rp >> 5;
    const int q = xw & (nq - 1);
    const int rb0 = xw / nq, rbs = TCC_XF_WARPS / nq;
    const int colpitchA = g.Rp * 16;
    const uint32_t thr = drop_threshold(op.p_elem);
    const float keep_s = op.p_elem > 0.f ? 1.0f / (1.0f - op.p_elem) : 1.f;
    const int raw_t = g.raw_tensor_bytes >> 2;
    for (int tile = blockIdx.x; tile < total && !*abort_s; tile += gridDim.x) {
      const int n = tile / tiles_per_n;
      const int p0 = (tile - n * tiles_per_n) * TCC_M - g.padA;
      float pfaf = 1.f;
      if (MODE == 1) pfaf = path_factor(op, seed, n) * alpha_factor(op, seed, n);
      for (int ch = 0; ch < g.nchunks; ++ch) {
        if (!tcc_wait(s32(&raw_full[rs]), rph, abort_s)) break;
        if (!tcc_wait(s32(&a_empty[as]), aph ^ 1, abort_s)) break;
        const float* raw = reinterpret_cast<const float*>(raw_s + (size_t)rs * g.n_raw * g.raw_tensor_bytes) + 4 * q * g.Rbox;
        unsigned char* a_hi = a_s + (size_t)as * g.a_stage + q * colpitchA;
        unsigned char* a_lo = a_hi + g.a_part;
        const int cbase = ch * g.KC + 4 * q;
        TccK e[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) e[j] = tk_s[cbase + j];
        const int nvalid = Kd - cbase;          // channels of this quad that exist (<= 0: padded quad, all zero)
        for (int rb = rb0; rb < nrb; rb += 2 * rbs) {
          // two 32-row blocks per iteration: 8 independent element chains in flight (the warps are latency-, not
          // throughput-bound otherwise), all shared-memory loads before the first store
          float t[2][4];
          int rrow[2];
          bool act[2];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = (rb + h * rbs) * 32 + lane;
            rrow[h] = r;
            act[h] = (rb + h * rbs) < nrb;
            const int p = p0 + r;
            const bool inb = act[h] && (r < g.R) && p >= 0 && p < g.src_len;
            const int rr = (act[h] && r < g.Rbox) ? r : 0;
            if (MODE == 0 && g.up) {
              // x2 linear up-sampling of f(source): position p = 2m takes 0.25 f(m-1) + 0.75 f(m), p = 2m+1 takes
              // 0.75 f(m) + 0.25 f(m+1), clamped at both ends (torch upsample_linear1d, align_corners=False)
              const int pc = p < 0 ? 0 : p;
              const int i0 = pc == 0 ? 0 : (pc - 1) >> 1;
              const int i1 = min(i0 + 1, g.up_S - 1);
              const float w1 = pc == 0 ? 0.f : ((pc & 1) ? 0.25f : 0.75f);
              const int s0 = tcc_up_src0(p0);
              const int a0 = min(max(i0 - s0, 0), g.Rbox - 1), a1 = min(max(i1 - s0, 0), g.Rbox - 1);
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                float f0 = fmaf(e[j].a, raw[j * g.Rbox + a0], e[j].b);
                float f1 = fmaf(e[j].a, raw[j * g.Rbox + a1], e[j].b);
                if (F_GELU && e[j].c != 0.f) { f0 = tcc_gelu(f0); f1 = tcc_gelu(f1); }
                const float v = fmaf(w1, f1 - f0, f0);
                t[h][j] = (inb && j < nvalid) ? v : 0.f;
              }
            } else if (MODE == 0) {
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                float v = fmaf(e[j].a, raw[j * g.Rbox + rr], e[j].b);
                if (F_GELU && e[j].c != 0.f) v = tcc_gelu(v);
                t[h][j] = (inb && j < nvalid) ? v : 0.f;
              }
            } else {
              uint64_t hq = 0ull;
              if (F_ELEM) {        // the 4 lanes of a sample quad share one hash per channel: each lane hashes ONE channel
                const int ck = min(cbase + (lane & 3), Kd - 1);
                hq = rng_u64(seed, op.seed_elem, (((uint64_t)n * op.Cout + ck) * (uint64_t)op.L_out + (uint64_t)(inb ? p : 0)) >> 2);
              }
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const int ro = j * g.Rbox + rr;
                int slot = 0;
                float dxd = 0.f, du = 0.f, x = 0.f;
                if (g.has_dxd) { dxd = raw[ro]; ++slot; }
                if (g.has_bn) { du = raw[slot * raw_t + ro]; ++slot; }
                if (g.need_x) { x = raw[slot * raw_t + ro]; }
                float gv = dxd + fmaf(e[j].a, du, fmaf(e[j].b, x, e[j].c));
                if (op.out_act == SEIST_OUT_SIGMOID) gv *= x * (1.f - x);
                gv *= pfaf;
                if (F_ELEM) {
                  const uint64_t hh = __shfl_sync(0xffffffffu, hq, (lane & ~3) | j);
                  gv *= (((uint32_t)(hh >> (16 * (p & 3))) & 0xFFFFu) >= thr) ? keep_s : 0.f;
                }
                t[h][j] = (inb && j < nvalid) ? gv : 0.f;
              }
            }
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (!act[h]) continue;
            float4 hi, lo;
            tcc_split(t[h][0], hi.x, lo.x);
            tcc_split(t[h][1], hi.y, lo.y);
            tcc_split(t[h][2], hi.z, lo.z);
            tcc_split(t[h][3], hi.w, lo.w);
            *reinterpret_cast<float4*>(a_hi + rrow[h] * 16) = hi;
            *reinterpret_cast<float4*>(a_lo + rrow[h] * 16) = lo;
          }
        }
        if (!g.b_resident) {
          unsigned char* bst = a_s + (size_t)as * g.a_stage + 2 * g.a_part;
          stage_b(ch, bst, bst + g.b_part, xw * 32 + lane, TCC_XF_WARPS * 32);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0) {
          tcc_arrive(s32(&a_full[as]));
          tcc_arrive(s32(&raw_empty[rs]));
        }
        if (++rs == g.raw_stages) { rs = 0; rph ^= 1; }
        if (++as == g.a_stages) { as = 0; aph ^= 1; }
      }
    }
  } else {
    // =========================== consumer warpgroups ===========================
    // warpgroup eg = warp / 4 multiplies rows 64 eg .. 64 eg + 63 of every tile into registers, both park their
    // accumulators in acc_s, then run the epilogue of the tile together: group eg takes the 16-channel chunks
    // c0 / 16 = eg (mod 2), warp % 4 a 32-row quadrant, lane = sample.  The tile loop does not test the abort flag, so
    // that both groups always meet at the named barriers; after an abort they only skip the work.
    const int eg = warp >> 2, wq = warp & 3;
    const int L = g.dst_len;
    const bool stats = MODE == 0 ? ((op.out.bn >= 0) && op.bn_table[op.out.bn >= 0 ? op.out.bn : 0].use_batch) : true;
    const float* ep_s = reinterpret_cast<const float*>(base + g.off_tab_n);
    const TccTgt* tg_s = reinterpret_cast<const TccTgt*>(base + g.off_tab_n);
    const uint32_t thr = drop_threshold(op.p_elem);
    const float keep_s = op.p_elem > 0.f ? 1.0f / (1.0f - op.p_elem) : 1.f;
    float* my_red = red_s + warp * 2 * Nd;
    const bool has_ra = MODE == 0 && op.res_a.C > 0, has_rb = MODE == 0 && op.res_b.C > 0;
    const bool sig = op.out_act == SEIST_OUT_SIGMOID;
    const size_t Ls = (size_t)L;
    const uint32_t colpitchA = (uint32_t)g.Rp * 16u;
    const int nq = g.KC >> 2;
    const int srow = 32 * wq + lane;                     // staged sample row this thread reads in the epilogue
    int as = 0;
    uint32_t aph = 0;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
      float acc[NB / 2];
      bool run = true;
      int prev = -1;                                     // stage whose MMAs may still be in flight
      for (int ch = 0; ch < g.nchunks; ++ch) {
        // issued whether or not the wait succeeded: a predicated wgmma serialises, and after an abort (bounded wait timed
        // out) the result of the tile is discarded anyway
        run = run && tcc_wait(s32(&a_full[as]), aph, abort_s);
        {
          const uint32_t a_hi = s32(a_s + (size_t)as * g.a_stage) + (uint32_t)(eg * 64 * 16);
          const uint32_t a_lo = a_hi + (uint32_t)g.a_part;
          uint32_t b_hi;
          if (g.b_resident) b_hi = s32(b_s + (size_t)ch * 2 * g.b_part);
          else b_hi = s32(a_s + (size_t)as * g.a_stage) + 2u * (uint32_t)g.a_part;
          const uint32_t b_lo = b_hi + (uint32_t)g.b_part;
          const int ksteps = min(g.KC, Kd - ch * g.KC + 7) >> 3;
          asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
          for (int t = 0; t < g.k; ++t) {
            for (int j = 0; j < ksteps; ++j) {
              const uint32_t aoff = (uint32_t)(2 * j) * colpitchA + (uint32_t)(t + g.toff) * 16u;
              const uint32_t boff = (uint32_t)(t * nq + 2 * j) * (uint32_t)colpitchB;
              const uint64_t ah = tcc_desc(a_hi + aoff, colpitchA, 128), al = tcc_desc(a_lo + aoff, colpitchA, 128);
              const uint64_t bh = tcc_desc(b_hi + boff, (uint32_t)colpitchB, 128), bl = tcc_desc(b_lo + boff, (uint32_t)colpitchB, 128);
              tcc_mma<NB>(acc, ah, bh, (ch > 0 || t > 0 || j > 0) ? 1u : 0u);
              tcc_mma<NB>(acc, al, bh, 1u);
              tcc_mma<NB>(acc, ah, bl, 1u);
            }
          }
          asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
          asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");   // the previous chunk's MMAs are done
        }
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) tcc_arrive(s32(&a_empty[prev]));   // this warp's reads of that stage are complete
        }
        prev = as;
        if (++as == g.a_stages) { as = 0; aph ^= 1; }
      }
      asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
      tcc_keep(acc);
      __syncwarp();
      if (lane == 0) tcc_arrive(s32(&a_empty[prev]));
      asm volatile("bar.sync 1, 256;" ::: "memory");    // the previous tile's epilogue is done with acc_s
      if (run) {
        const int r0 = eg * 64 + wq * 16 + (lane >> 2);
        const int cl = 2 * (lane & 3);
#pragma unroll
        for (int e = 0; e < NB / 2; ++e)
          acc_s[(8 * (e >> 2) + cl + (e & 1)) * TCC_ACC_PITCH + r0 + 8 * ((e >> 1) & 1)] = acc[e];
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (!run || *abort_s) continue;
      const int n = tile / tiles_per_n;
      const int l = (tile - n * tiles_per_n) * TCC_M + srow;
      const bool ok = l < L;
      const int ls = ok ? l : 0;
      if (MODE == 0) {
        const float pf = path_factor(op, seed, n), af = alpha_factor(op, seed, n);
        float* optr = op.out.x + ((size_t)n * op.out.Ct + op.out.c0 + 16 * eg) * Ls + ls;
        const float* ra = has_ra ? op.res_a.x + ((size_t)n * op.res_a.Ct + op.res_a.c0 + 16 * eg) * Ls + ls : nullptr;
        const float* rb = has_rb ? op.res_b.x + ((size_t)n * op.res_b.Ct + op.res_b.c0 + 16 * eg) * Ls + ls : nullptr;
#pragma unroll 1
        for (int c0 = 16 * eg; c0 < Nd; c0 += 32) {
          uint32_t rr[16];
          TCC_LD16(rr, c0);
          const int nv = min(16, Nd - c0);               // uniform
          float val[16];
#pragma unroll
          for (int c = 0; c < 16; ++c) val[c] = (__uint_as_float(rr[c]) + ep_s[min(c0 + c, Nd - 1)]) * pf;
          if (F_ELEM) {
#pragma unroll
            for (int qd = 0; qd < 4; ++qd) {
              const int ck = min(c0 + 4 * qd + (lane & 3), Nd - 1);
              const uint64_t hq = rng_u64(seed, op.seed_elem, (((uint64_t)n * Nd + ck) * (uint64_t)L + (uint64_t)ls) >> 2);
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const uint64_t hh = __shfl_sync(0xffffffffu, hq, (lane & ~3) | j);
                val[4 * qd + j] *= ((uint32_t)(hh >> (16 * (l & 3))) & 0xFFFFu) >= thr ? keep_s : 0.f;
              }
            }
          }
          if (has_ra) {
            float rv[16];
#pragma unroll
            for (int c = 0; c < 16; ++c) rv[c] = __ldg(ra + (size_t)min(c, nv - 1) * Ls);
#pragma unroll
            for (int c = 0; c < 16; ++c) val[c] += fmaf(ep_s[Nd + min(c0 + c, Nd - 1)], rv[c], ep_s[2 * Nd + min(c0 + c, Nd - 1)]);
            ra += 32 * Ls;
          }
          if (af != 1.f) {
#pragma unroll
            for (int c = 0; c < 16; ++c) val[c] *= af;
          }
          if (has_rb) {
            float rv[16];
#pragma unroll
            for (int c = 0; c < 16; ++c) rv[c] = __ldg(rb + (size_t)min(c, nv - 1) * Ls);
#pragma unroll
            for (int c = 0; c < 16; ++c) val[c] += fmaf(ep_s[3 * Nd + min(c0 + c, Nd - 1)], rv[c], ep_s[4 * Nd + min(c0 + c, Nd - 1)]);
            rb += 32 * Ls;
          }
          if (sig) {
#pragma unroll
            for (int c = 0; c < 16; ++c) val[c] = sigmoid_f(val[c]);
          }
          float* op_c = optr;
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            const bool w = ok && c < nv;
            if (w) *op_c = val[c];
            val[c] = w ? val[c] : 0.f;
            op_c += Ls;
          }
          optr += 32 * Ls;
          if (stats) {
            float s2[16];
#pragma unroll
            for (int c = 0; c < 16; ++c) s2[c] = val[c] * val[c];
            const float t1 = tcc_reduce16(val, lane), t2 = tcc_reduce16(s2, lane);
            const int co = c0 + tcc_red_index(lane);
            if ((lane & 1) == 0 && co < Nd) {        // single writer per (warp, channel): deterministic
              my_red[2 * co] += t1;
              my_red[2 * co + 1] += t2;
            }
          }
        }
      } else {
#pragma unroll 1
        for (int c0 = 16 * eg; c0 < Nd; c0 += 32) {
          uint32_t rr[16];
          TCC_LD16(rr, c0);
          float xv[16], ov[16];
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            const TccTgt& e = tg_s[min(c0 + c, Nd - 1)];
            const bool live = ok && (c0 + c < Nd) && e.g != nullptr;
            const long long off = (long long)n * e.nstride + ls;
            xv[c] = (live && (e.bn >= 0 || (F_GELU && e.act == SEIST_ACT_GELU))) ? __ldg(e.x + off) : 0.f;
            ov[c] = (live && e.accum) ? e.g[off] : 0.f;
          }
          float s1[16], s2[16];
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            const TccTgt& e = tg_s[min(c0 + c, Nd - 1)];
            const bool live = ok && (c0 + c < Nd) && e.g != nullptr;
            float gg = live ? __uint_as_float(rr[c]) : 0.f;
            if (F_GELU && e.act == SEIST_ACT_GELU) gg *= tcc_gelu_grad(fmaf(e.sc, xv[c], e.sh));
            const bool st = live && e.bn >= 0;
            s1[c] = st ? gg : 0.f;
            s2[c] = st ? gg * ((xv[c] - e.mu) * e.istd) : 0.f;
            if (live) e.g[(long long)n * e.nstride + l] = gg + ov[c];
          }
          const float t1 = tcc_reduce16(s1, lane), t2 = tcc_reduce16(s2, lane);
          const int ci = c0 + tcc_red_index(lane);
          if ((lane & 1) == 0 && ci < Nd) {
            my_red[2 * ci] += t1;
            my_red[2 * ci + 1] += t2;
          }
        }
      }
    }
  }

  // ---- teardown ---------------------------------------------------------------------------------------------------
  __syncthreads();
  if (MODE == 0) {
    const bool stats = (op.out.bn >= 0) && op.bn_table[op.out.bn >= 0 ? op.out.bn : 0].use_batch;
    if (stats) {
      const SeistBN& e = op.bn_table[op.out.bn];
      for (int i = tid; i < 2 * Nd; i += TCC_NT) {
        float s = 0.f;
        for (int w = 0; w < TCC_EPI_WARPS; ++w) s += red_s[w * 2 * Nd + i];
        atomicAdd(&e.stat_acc[(i & 1) * e.C + op.out.bn_c0 + (i >> 1)], (double)s);
      }
    }
  } else {
    const TccTgt* tg_s = reinterpret_cast<const TccTgt*>(base + g.off_tab_n);
    for (int i = tid; i < 2 * Nd; i += TCC_NT) {
      const TccTgt& t = tg_s[i >> 1];
      if (t.g != nullptr && t.bn >= 0) {
        float s = 0.f;
        for (int w = 0; w < TCC_EPI_WARPS; ++w) s += red_s[w * 2 * Nd + i];
        const SeistBN& e = op.bn_table[t.bn];
        atomicAdd(&e.gstat_acc[(i & 1) * e.C + t.bnc], (double)s);
      }
    }
  }
  if (tid == 0 && *abort_s) atomicExch(&g_tcc_err_dev, 1);
}

// ================================================================================================================
// host side
// ================================================================================================================
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn tcc_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// (N, Ct, L) fp32 tensor -> 3-D map with box {rows, 8 channels, 1 waveform}
static int tcc_make_map(CUtensorMap* m, const float* basep, int L, int Ct, int N, int box_rows) {
  EncodeTiledFn fn = tcc_encode_fn();
  if (!fn) { set_error("tcconv: cuTensorMapEncodeTiled unavailable"); return -3; }
  const cuuint64_t dims[3] = {(cuuint64_t)L, (cuuint64_t)Ct, (cuuint64_t)N};
  const cuuint64_t strides[2] = {(cuuint64_t)L * 4ull, (cuuint64_t)L * (cuuint64_t)Ct * 4ull};
  const cuuint32_t box[3] = {(cuuint32_t)box_rows, 8u, 1u};
  const cuuint32_t estr[3] = {1u, 1u, 1u};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(basep), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("tcconv: cuTensorMapEncodeTiled failed"); return -3; }
  return 0;
}


bool tcconv_eligible(const SeistOp& op, int mode) {
  if (op.stride != 1 || op.pool > 1 || op.k > 32) return false;
  if ((mode == 0 ? op.Cout : op.Cin) > TCC_NMAX) return false;   // accumulator registers of the consumer warpgroups
  if (op.L_in != op.L_out || (op.L_out & 3)) return false;       // TMA: 16-byte row pitch
  if (op.up_src_L > 0) {     // x2 linear up-sampling folded into the forward transform (the dpk head, models/seist.py:560-566)
    if (mode != 0 || op.n_in != 1 || op.L_in != 2 * op.up_src_L || (op.up_src_L & 3) || op.in[0].L != op.up_src_L) return false;
    return (reinterpret_cast<uintptr_t>(op.in[0].x) & 15) == 0;
  }
  if (op.Cout > 256 || op.Cin > 256) return false;
  if (op.k > 1 && op.p_elem > 0.f) return false;                 // quad-aligned dropout hashing assumes l0 % 4 == 0 rows
  for (int i = 0; i < op.n_in; ++i) {
    if (op.in[i].L != op.L_in) return false;
    if (op.n_in > 1 && (op.in[i].C & 7)) return false;          // TMA boxes of 8 channels must not straddle views
    if ((reinterpret_cast<uintptr_t>(op.in[i].x) & 15) != 0) return false;
  }
  if (mode == 1) {
    bool any = false;
    for (int i = 0; i < op.n_in; ++i) any = any || op.in[i].g != nullptr;
    if (!any) return false;
    if ((reinterpret_cast<uintptr_t>(op.out.x) & 15) != 0) return false;
  }
  return true;
}

static bool tcc_geometry(const SeistOp& op, int mode, TccGeom& g) {
  g = TccGeom{};
  g.mode = mode;
  g.Kd = mode == 0 ? op.Cin : op.Cout;
  g.Nd = mode == 0 ? op.Cout : op.Cin;
  g.k = op.k;
  g.padl = mode == 0 ? op.pad_left : op.k - 1 - op.pad_left;
  g.src_len = mode == 0 ? op.L_in : op.L_out;
  g.dst_len = mode == 0 ? op.L_out : op.L_in;
  g.padA = (g.padl + 3) & ~3;
  g.toff = g.padA - g.padl;
  g.R = TCC_M + op.k - 1 + g.toff;
  g.up = (mode == 0 && op.up_src_L > 0) ? 1 : 0;
  g.up_S = op.up_src_L;
  g.Rbox = g.up ? ((g.R / 2 + 6 + 3) & ~3) : ((g.R + 3) & ~3);       // raw rows staged per tile (source rows when up-sampling)
  g.Rp = (g.R + 31) & ~31;
  g.N_pad = g.Nd <= 32 ? 32 : (g.Nd <= 64 ? 64 : 128);
  if (g.N_pad > TCC_NMAX) return false;
  const bool has_bn = (op.out.bn >= 0 && op.out.g != nullptr);
  g.has_dxd = (mode == 1 && op.out_dxd != nullptr) ? 1 : 0;
  g.has_bn = (mode == 1 && has_bn) ? 1 : 0;
  g.need_x = (mode == 1 && (has_bn || op.out_act == SEIST_OUT_SIGMOID)) ? 1 : 0;
  g.n_raw = mode == 0 ? 1 : g.has_dxd + g.has_bn + g.need_x;
  if (g.n_raw == 0) return false;
  const int tab_n = mode == 0 ? 5 * g.Nd * 4 : g.Nd * (int)sizeof(TccTgt);
  const int budget = 220 * 1024;
  // chunk width: fewest padded reduction channels first (the transform warps pay for padding), wider chunks second
  int kcs[3] = {32, 16, 8};
  {
    const int k8 = (g.Kd + 7) & ~7;
    auto waste = [&](int kc) { return ((k8 + kc - 1) / kc) * kc - k8; };
    for (int i = 0; i < 3; ++i)
      for (int j = i + 1; j < 3; ++j)
        if (waste(kcs[j]) < waste(kcs[i])) { const int tmp = kcs[i]; kcs[i] = kcs[j]; kcs[j] = tmp; }
  }
  for (int resident = 1; resident >= 0; --resident) {
    for (int ki = 0; ki < 3; ++ki) {
      const int KC = kcs[ki];
      g.KC = KC;
      g.nchunks = (g.Kd + KC - 1) / KC;
      g.raw_tensor_bytes = KC * g.Rbox * 4;
      g.a_part = (KC / 4) * g.Rp * 16;
      g.b_part = g.k * (KC / 4) * g.N_pad * 16;
      g.b_resident = resident;
      const int b_bytes = resident ? g.nchunks * 2 * g.b_part : 0;
      const int a_stage = 2 * g.a_part + (resident ? 0 : 2 * g.b_part);
      g.a_stage = a_stage;
      const int raw_stage = g.n_raw * g.raw_tensor_bytes;
      const int acc_bytes = g.N_pad * TCC_ACC_PITCH * 4;
      const int fixed = b_bytes + g.nchunks * KC * (int)sizeof(TccK) + tab_n + 16 * g.Nd * 4 + acc_bytes + 4 * TCC_MAX_STAGES * 8 + 64 + 256;
      for (int st = 4; st >= 2; --st) {
        const int rst = st + 1 > TCC_MAX_STAGES ? TCC_MAX_STAGES : st + 1;
        const int tot = fixed + st * a_stage + rst * raw_stage;
        if (tot <= budget) {
          g.a_stages = st;
          g.raw_stages = rst;
          int off = 0;
          g.off_raw = off; off += rst * raw_stage;
          g.off_a = off; off += st * a_stage;
          g.off_b = off; off += b_bytes;
          g.off_tab_k = off; off += g.nchunks * KC * (int)sizeof(TccK);
          off = (off + 15) & ~15;
          g.off_tab_n = off; off += tab_n;
          off = (off + 15) & ~15;
          g.off_red = off; off += 16 * g.Nd * 4;
          off = (off + 15) & ~15;
          g.off_acc = off; off += acc_bytes;
          g.off_bar = off; off += 4 * TCC_MAX_STAGES * 8 + 64;
          g.smem_bytes = off + 128;
          return true;
        }
      }
    }
  }
  return false;
}

template <int MODE, bool G, bool E, int NB>
static int tcc_go_nb(const SeistOp& op, const TccGeom& g, const TccMaps& maps, unsigned grid, cudaStream_t s) {
  static bool attr_set[64] = {false};        // the attribute is per device
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr_set[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(tcconv_kernel<MODE, G, E, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); return (int)e; }
    attr_set[dev & 63] = true;
  }
  tcconv_kernel<MODE, G, E, NB><<<grid, TCC_NT, g.smem_bytes, s>>>(op, g, maps);
  return 0;
}
template <int MODE, bool G, bool E>
static int tcc_go(const SeistOp& op, const TccGeom& g, const TccMaps& maps, unsigned grid, cudaStream_t s) {
  if (g.N_pad == 32) return tcc_go_nb<MODE, G, E, 32>(op, g, maps, grid, s);
  if (g.N_pad == 64) return tcc_go_nb<MODE, G, E, 64>(op, g, maps, grid, s);
  return tcc_go_nb<MODE, G, E, 128>(op, g, maps, grid, s);
}

int launch_tcconv(const SeistOp& op, int mode, cudaStream_t s, int sm_count) {
  TccGeom g;
  if (!tcc_geometry(op, mode, g)) { set_error("tcconv: no shared-memory configuration"); return -2; }
  TccMaps maps;
  std::memset(&maps, 0, sizeof(maps));
  int rc = 0;
  if (mode == 0) {
    for (int i = 0; i < op.n_in && !rc; ++i) rc = tcc_make_map(&maps.m[i], op.in[i].x, op.in[i].L, op.in[i].Ct, op.N, g.Rbox);
  } else {
    if (g.has_dxd) rc = tcc_make_map(&maps.m[0], op.out_dxd, op.out.L, op.out.Ct, op.N, g.Rbox);
    if (!rc && g.has_bn) rc = tcc_make_map(&maps.m[1], op.out.g, op.out.L, op.out.Ct, op.N, g.Rbox);
    if (!rc && g.need_x) rc = tcc_make_map(&maps.m[2], op.out.x, op.out.L, op.out.Ct, op.N, g.Rbox);
  }
  if (rc) return rc;
  const long tiles = (long)op.N * ((g.dst_len + TCC_M - 1) / TCC_M);
  long gr = sm_count;
  if (gr > tiles) gr = tiles;
  const unsigned grid = (unsigned)(gr < 1 ? 1 : gr);
  bool gelu = false;
  for (int i = 0; i < op.n_in; ++i) gelu = gelu || op.in[i].act == SEIST_ACT_GELU;
  const bool elem = op.p_elem > 0.f;
  if (mode == 0) {
    if (gelu) rc = elem ? tcc_go<0, true, true>(op, g, maps, grid, s) : tcc_go<0, true, false>(op, g, maps, grid, s);
    else rc = elem ? tcc_go<0, false, true>(op, g, maps, grid, s) : tcc_go<0, false, false>(op, g, maps, grid, s);
  } else {
    if (gelu) rc = elem ? tcc_go<1, true, true>(op, g, maps, grid, s) : tcc_go<1, true, false>(op, g, maps, grid, s);
    else rc = elem ? tcc_go<1, false, true>(op, g, maps, grid, s) : tcc_go<1, false, false>(op, g, maps, grid, s);
  }
  if (rc) return rc;
  note_launch();
  return check_launch(mode == 0 ? "tcconv_fwd" : "tcconv_bwd_data");
}

int tcconv_error_flag() {
  int v = 0;
  cudaMemcpyFromSymbol(&v, g_tcc_err_dev, sizeof(int));
  return v;
}

}  // namespace seist
