// Pointwise (k = 1, stride 1, groups 1) convolutions — the bulk of the encoder FLOPs and bytes
// (reference models/seist.py:86,107,111,130,142,182,225,287,351-364,429,451).
//
// Streaming design: a thread owns one quad of 4 consecutive samples and a tile of output channels; it
// walks the reduction channels 8 at a time, issuing eight independent 16-byte global loads before any
// use (memory-level parallelism instead of a staged tile), applies BatchNorm/GELU of the consumer view in
// registers and accumulates against weights held k-major in shared memory (one broadcast vector per
// reduction channel).  A CTA runs G quads per thread back to back so the BatchNorm statistics of the
// result are carried in registers and reduced (shuffles -> shared -> one double atomic per channel) once.
#include "common.cuh"
#include "conv_common.cuh"

namespace seist {

constexpr int PW_NT = 128;

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// per-thread asynchronous copy ring (LDGSTS, helpers in common.cuh): a thread copies ITS OWN 16-byte operands global ->
// shared several contraction steps ahead and reads them back from the same slot: no registers are held while the loads
// are in flight and no cross-thread synchronisation is needed (cp.async.wait_group orders the issuing thread's own copies).
__device__ __forceinline__ float4 lds4(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
  return v;
}

struct PwChan {          // one reduction / target channel, resolved once per CTA
  const float* x;        // row base for n = 0
  float* g;              // gradient row base for n = 0 (backward targets) or nullptr
  long long nstride;     // elements between consecutive waveforms
  float sc, sh, mu, istd;
  int act, bn, bnc, accum;
};

__device__ __forceinline__ PwChan make_chan(const SeistOp& op, int ci, bool want_khat) {
  int cv;
  const int vi = resolve_view(op, ci, cv);
  const SeistView& v = op.in[vi];
  PwChan c;
  c.x = v.x + (size_t)(v.c0 + cv) * v.L;
  c.g = v.g ? v.g + (size_t)(v.c0 + cv) * v.L : nullptr;
  c.nstride = (long long)v.Ct * v.L;
  view_coef(op, v, cv, c.sc, c.sh);
  c.mu = 0.f;
  c.istd = 0.f;
  if (want_khat && v.bn >= 0) view_khat(op, v, cv, c.mu, c.istd);
  c.act = v.act;
  c.bn = v.bn;
  c.bnc = v.bn_c0 + cv;
  c.accum = v.accum;
  return c;
}

// (scalar on purpose: the latency-bound 1x1 kernels interleave this math with their loads; the staged kernels, where the
// transform is a separate pass over shared memory, use the two-lane forms)
__device__ __forceinline__ float4 apply_view(float4 v, float sc, float sh, int act) {
  v.x = fmaf(sc, v.x, sh);
  v.y = fmaf(sc, v.y, sh);
  v.z = fmaf(sc, v.z, sh);
  v.w = fmaf(sc, v.w, sh);
  if (act == SEIST_ACT_GELU) {
    v.x = gelu_f(v.x);
    v.y = gelu_f(v.y);
    v.z = gelu_f(v.z);
    v.w = gelu_f(v.w);
  }
  return v;
}
// packed variant for the staging passes of the weight-gradient kernel
__device__ __forceinline__ float4 apply_view2(float4 v, float sc, float sh, int act) {
  v = affine4(v, sc, sh);
  if (act == SEIST_ACT_GELU) v = gelu4(v);
  return v;
}

// ---- pooled consumer view (reference LAAB / KV aggregation: AvgPool1d(P) + MaxPool1d(P), models/seist.py:62-76) ----
// the 4 pooled samples l..l+3 of a channel come from the 4*P contiguous source samples starting at l*P
__device__ __forceinline__ float pool_pair(float a, float b) { return 0.5f * (a + b) + fmaxf(a, b); }
__device__ __forceinline__ float4 pw_load_pooled(const float* src, int P, float sc, float sh) {
  float4 r;
  if (P == 2) {
    const float4 a = apply_view(ldg4(src), sc, sh, 0), b = apply_view(ldg4(src + 4), sc, sh, 0);
    r = make_float4(pool_pair(a.x, a.y), pool_pair(a.z, a.w), pool_pair(b.x, b.y), pool_pair(b.z, b.w));
  } else {
    const int QP = P >> 2;   // float4 per pooled sample (P = 4, 8)
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float sum = 0.f, mx = -INFINITY;
      for (int i = 0; i < QP; ++i) {
        const float4 a = apply_view(ldg4(src + 4 * (j * QP + i)), sc, sh, 0);
        sum += (a.x + a.y) + (a.z + a.w);
        mx = fmaxf(fmaxf(mx, fmaxf(a.x, a.y)), fmaxf(a.z, a.w));
      }
      o[j] = sum / (float)P + mx;
    }
    r = make_float4(o[0], o[1], o[2], o[3]);
  }
  return r;
}

// Backward of AvgPool1d(P) + MaxPool1d(P) in front of a 1x1 conv (reference models/seist.py:62-76) for one target channel
// of one thread: NJ pooled gradients gq[0..NJ) go to their NJ*P contiguous source samples as g * (1/P + [first arg max of the
// BN-applied values]).  The source samples are read and written with 16-byte accesses and the arg max is found in
// registers instead of P scalar loads + P/2 float2 loads and stores per pooled sample.  s1 / s2: BN-backward sums of the targets.
template <int P, int NJ>
__device__ __forceinline__ void pool_route_part(const PwChan& c, const float4* xs, float4* gs, const float* gq, float& s1,
                                                float& s2) {
  constexpr int NC = NJ * P / 4;                 // float4 chunks
  constexpr float invp = 1.f / (float)P;
  float v[NJ * P];
#pragma unroll
  for (int k = 0; k < NC; ++k) {
    const float4 q = __ldg(xs + k);
    v[4 * k] = q.x;
    v[4 * k + 1] = q.y;
    v[4 * k + 2] = q.z;
    v[4 * k + 3] = q.w;
  }
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    int am = 0;
    float mx = fmaf(c.sc, v[j * P], c.sh);
#pragma unroll
    for (int i = 1; i < P; ++i) {
      const float u = fmaf(c.sc, v[j * P + i], c.sh);
      if (u > mx) {
        mx = u;
        am = i;
      }
    }
#pragma unroll
    for (int i = 0; i < P; ++i) {
      const float x = v[j * P + i];
      const float g = gq[j] * (invp + (i == am ? 1.f : 0.f));
      s1 += g;
      s2 = fmaf(g, (x - c.mu) * c.istd, s2);
      v[j * P + i] = g;
    }
  }
  if (c.accum) {
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      const float4 o = gs[k];
      v[4 * k] += o.x;
      v[4 * k + 1] += o.y;
      v[4 * k + 2] += o.z;
      v[4 * k + 3] += o.w;
    }
  }
#pragma unroll
  for (int k = 0; k < NC; ++k) gs[k] = make_float4(v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]);
}
template <int P>
__device__ __forceinline__ void pool_route(const PwChan& c, long long soff, float4 gg, float& s1, float& s2) {
  const float4* xs = reinterpret_cast<const float4*>(c.x + soff);
  float4* gs = reinterpret_cast<float4*>(c.g + soff);
  const float gq[4] = {gg.x, gg.y, gg.z, gg.w};
  if constexpr (P == 8) {      // two halves: 16 source samples in registers at a time
    pool_route_part<8, 2>(c, xs, gs, gq, s1, s2);
    pool_route_part<8, 2>(c, xs + 4, gs + 4, gq + 2, s1, s2);
  } else {
    pool_route_part<P, 4>(c, xs, gs, gq, s1, s2);
  }
}

// CTA-wide reduction of per-thread partial sums part[NV] -> double atomics.  red_s: [4][NV] floats.
template <int NV, typename F>
__device__ __forceinline__ void cta_reduce_atomic(float (&part)[NV], float* red_s, F&& sink) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float s = warp_sum(part[i]);
    if (lane == 0) red_s[warp * NV + i] = s;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < NV; i += PW_NT) {
    const float s = red_s[i] + red_s[NV + i] + red_s[2 * NV + i] + red_s[3 * NV + i];
    sink(i, s);
  }
}

// ================================================================================================
// forward: out[co] = alpha * [ drop( sum_ci W[co][ci] f(in[ci]) + b ) + res_a ] + res_b
// grid (ceil(N*L/4 / (128*G)), ceil(Cout/COUT_T))
// ================================================================================================
__device__ __noinline__ float4 pw_gelu4(float4 v) {
  v.x = gelu_f(v.x);
  v.y = gelu_f(v.y);
  v.z = gelu_f(v.z);
  v.w = gelu_f(v.w);
  return v;
}
__device__ __noinline__ float4 pw_gelu_grad4(float4 u) {
  u.x = gelu_grad_f(u.x);
  u.y = gelu_grad_f(u.y);
  u.z = gelu_grad_f(u.z);
  u.w = gelu_grad_f(u.w);
  return u;
}
__device__ __noinline__ float4 pw_keep4(float p, uint64_t seed, uint32_t stream, uint64_t idx) {
  return keep4(p, seed, stream, idx);
}

// compile-time specialisation keeps the bodies small (instruction cache) and the inner loops free of
// runtime feature tests: F_ELEM element dropout, F_RES residual views, F_GELU some view applies GELU
template <int COUT_T, bool F_ELEM, bool F_RES, bool F_GELU, bool F_POOL = false>
__global__ void __launch_bounds__(PW_NT, 4) pw_fwd_kernel(const __grid_constant__ SeistOp op, const int G) {
  extern __shared__ __align__(16) unsigned char sm_raw[];
  const int Cin = op.Cin, Cin8 = (Cin + 7) & ~7;
  PwChan* ch_s = reinterpret_cast<PwChan*>(sm_raw);                       // [Cin8]
  float* w_s = reinterpret_cast<float*>(ch_s + Cin8);                     // [Cin8][COUT_T]
  float* ep_s = w_s + Cin8 * COUT_T;                                      // bias, ra_sc, ra_sh, rb_sc, rb_sh [COUT_T] each
  float* red_s = ep_s + 5 * COUT_T;                                       // [4][2*COUT_T]
  float* st_s = red_s + 4 * 2 * COUT_T;                                   // [4 warps][2*COUT_T][32 lanes] running sums
  const int tid = threadIdx.x;
  const int co_base = blockIdx.y * COUT_T;
  const int L = op.L_out, LQ = L >> 2;

  for (int ci = tid; ci < Cin8; ci += PW_NT) {
    if (ci < Cin) {
      ch_s[ci] = make_chan(op, ci, false);
    } else {
      PwChan z = make_chan(op, 0, false);
      z.act = 0;
      ch_s[ci] = z;   // padded channel: valid address, zero weights
    }
  }
  for (int idx = tid; idx < Cin8 * COUT_T; idx += PW_NT) {
    const int ci = idx / COUT_T, col = idx - ci * COUT_T;
    const int co = co_base + col;
    w_s[idx] = (co < op.Cout && ci < Cin) ? op.W[(size_t)co * Cin + ci] : 0.f;
  }
  for (int col = tid; col < COUT_T; col += PW_NT) {
    const int co = co_base + col;
    float b = 0.f, asc = 1.f, ash = 0.f, bsc = 1.f, bsh = 0.f;
    if (co < op.Cout) {
      if (op.bias) b = op.bias[co];
      if (op.res_a.C > 0) view_coef(op, op.res_a, co, asc, ash);
      if (op.res_b.C > 0) view_coef(op, op.res_b, co, bsc, bsh);
    }
    ep_s[col] = b;
    ep_s[COUT_T + col] = asc;
    ep_s[2 * COUT_T + col] = ash;
    ep_s[3 * COUT_T + col] = bsc;
    ep_s[4 * COUT_T + col] = bsh;
  }
  __syncthreads();

  const uint64_t seed = load_seed(op.step_seed);
  const long long NQ = (long long)op.N * LQ;
  const bool stats = (op.out.bn >= 0) && op.bn_table[op.out.bn >= 0 ? op.out.bn : 0].use_batch;
  // BatchNorm sums of the result live in shared memory (one private slot per thread and statistic) between
  // quads: in registers they would cost 2*COUT_T registers across the whole contraction loop
  float* my_st = st_s + (tid >> 5) * (2 * COUT_T * 32) + (tid & 31);
#pragma unroll
  for (int i = 0; i < 2 * COUT_T; ++i) my_st[i * 32] = 0.f;

  for (int g = 0; g < G; ++g) {
    const long long f = ((long long)blockIdx.x * G + g) * PW_NT + tid;
    const bool ok = f < NQ;
    const int n = ok ? (int)(f / LQ) : 0;
    const int l = ok ? (int)(f - (long long)n * LQ) * 4 : 0;
    float2 acc[COUT_T / 2][4];   // [channel pair][sample]: .x = even channel, .y = odd channel (fma2 lanes)
#pragma unroll
    for (int c = 0; c < COUT_T / 2; ++c)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[c][q] = make_float2(0.f, 0.f);
    for (int ci0 = 0; ci0 < Cin8; ci0 += 8) {
      float4 v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const PwChan& c = ch_s[ci0 + j];
        if (F_POOL) v[j] = pw_load_pooled(c.x + (long long)n * c.nstride + (long long)l * op.pool, op.pool, c.sc, c.sh);
        else v[j] = ldg4(c.x + (long long)n * c.nstride + l);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const PwChan& c = ch_s[ci0 + j];
        float4 u = F_POOL ? v[j] : apply_view(v[j], c.sc, c.sh, 0);
        if (F_GELU && c.act == SEIST_ACT_GELU) u = pw_gelu4(u);
        const float2* wr = reinterpret_cast<const float2*>(w_s + (ci0 + j) * COUT_T);
        const float2 ux = dup2(u.x), uy = dup2(u.y), uz = dup2(u.z), uw = dup2(u.w);
#pragma unroll
        for (int cp = 0; cp < COUT_T / 2; ++cp) {
          const float2 w = wr[cp];
          acc[cp][0] = fma2(w, ux, acc[cp][0]);
          acc[cp][1] = fma2(w, uy, acc[cp][1]);
          acc[cp][2] = fma2(w, uz, acc[cp][2]);
          acc[cp][3] = fma2(w, uw, acc[cp][3]);
        }
      }
    }
    if (!ok) continue;
    const float pf = path_factor(op, seed, n), af = alpha_factor(op, seed, n);
    // output channels in batches of 4: the residual loads of a batch are issued before its first store (the
    // compiler cannot move loads across possibly aliasing stores, which serialised load -> use -> store per channel)
#pragma unroll
    for (int cb = 0; cb < COUT_T; cb += 4) {
      float4 ra[4], rb[4];
      if (F_RES) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int co = min(co_base + cb + u, op.Cout - 1);
          ra[u] = op.res_a.C > 0 ? ldg4(op.res_a.x + ((size_t)n * op.res_a.Ct + op.res_a.c0 + co) * (size_t)L + l)
                                 : make_float4(0.f, 0.f, 0.f, 0.f);
          rb[u] = op.res_b.C > 0 ? ldg4(op.res_b.x + ((size_t)n * op.res_b.Ct + op.res_b.c0 + co) * (size_t)L + l)
                                 : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int col = cb + u;
        const int co = co_base + col;
        if (co >= op.Cout) break;
        const float2(&ap)[4] = acc[col >> 1];
        float4 r = (col & 1) ? make_float4(ap[0].y, ap[1].y, ap[2].y, ap[3].y) : make_float4(ap[0].x, ap[1].x, ap[2].x, ap[3].x);
        const float b = ep_s[col];
        r.x = (r.x + b) * pf;
        r.y = (r.y + b) * pf;
        r.z = (r.z + b) * pf;
        r.w = (r.w + b) * pf;
        if (F_ELEM) {
          const float4 kp = pw_keep4(op.p_elem, seed, op.seed_elem, ((uint64_t)n * op.Cout + co) * (uint64_t)L + l);
          r.x *= kp.x;
          r.y *= kp.y;
          r.z *= kp.z;
          r.w *= kp.w;
        }
        if (F_RES && op.res_a.C > 0) {
          const float4 a = ra[u];
          const float sc = ep_s[COUT_T + col], sh = ep_s[2 * COUT_T + col];
          r.x += fmaf(sc, a.x, sh);
          r.y += fmaf(sc, a.y, sh);
          r.z += fmaf(sc, a.z, sh);
          r.w += fmaf(sc, a.w, sh);
        }
        r.x *= af;
        r.y *= af;
        r.z *= af;
        r.w *= af;
        if (F_RES && op.res_b.C > 0) {
          const float4 a = rb[u];
          const float sc = ep_s[3 * COUT_T + col], sh = ep_s[4 * COUT_T + col];
          r.x += fmaf(sc, a.x, sh);
          r.y += fmaf(sc, a.y, sh);
          r.z += fmaf(sc, a.z, sh);
          r.w += fmaf(sc, a.w, sh);
        }
        if (op.out_act == SEIST_OUT_SIGMOID) {
          r.x = sigmoid_f(r.x);
          r.y = sigmoid_f(r.y);
          r.z = sigmoid_f(r.z);
          r.w = sigmoid_f(r.w);
        }
        st4(op.out.x + ((size_t)n * op.out.Ct + op.out.c0 + co) * (size_t)L + l, r);
        if (stats) {
          my_st[(2 * col) * 32] += (r.x + r.y) + (r.z + r.w);
          my_st[(2 * col + 1) * 32] += fmaf(r.x, r.x, r.y * r.y) + fmaf(r.z, r.z, r.w * r.w);
        }
      }
    }
  }
  if (stats) {
    float st[2 * COUT_T];
#pragma unroll
    for (int i = 0; i < 2 * COUT_T; ++i) st[i] = my_st[i * 32];
    cta_reduce_atomic<2 * COUT_T>(st, red_s, [&](int i, float s) {
      const int co = co_base + (i >> 1);
      if (co < op.Cout) {
        const SeistBN& e = op.bn_table[op.out.bn];
        atomicAdd(&e.stat_acc[(i & 1) * e.C + op.out.bn_c0 + co], (double)s);
      }
    });
  }
}

// ================================================================================================
// backward (data): d in[ci] = sum_co W[co][ci] gacc[co];  gacc = dOut * alpha * delta * D
// dOut = A*du + Bx*x + Cc + dxd (then sigmoid').  grid (ceil(NQ/(128*G)), ceil(Cin/CI_T))
// ================================================================================================
constexpr int PW_BD_EB = 4;   // target channels whose epilogue loads are issued together
constexpr int PW_BD_CG = 2;   // output channels whose gradient loads are in flight together (register budget: 4 CTAs/SM)
struct PwOut {   // per output channel of the forward op, resolved once per CTA
  float A, Bx, Cc;
};

constexpr int PW_RING_S = 3;                                   // ring stages (PW_RING_S - 1 contraction steps in flight)
constexpr int PW_RING_STAGE_B = PW_BD_CG * 3 * PW_NT * 16;     // bytes per stage: [channel][dxd | du | x][thread] float4
template <int CI_T, bool F_ELEM, bool F_GELU, bool F_POOL = false>
__global__ void __launch_bounds__(PW_NT, 4) pw_bwd_data_kernel(const __grid_constant__ SeistOp op, const int G) {
  constexpr bool RING = !F_POOL;   // the pooled instantiation loads its operands directly
  extern __shared__ __align__(16) unsigned char sm_raw[];
  const int Cout = op.Cout, Cout4 = (Cout + 3) & ~3, Cin = op.Cin;
  PwChan* ch_s = reinterpret_cast<PwChan*>(sm_raw);                       // [CI_T] targets
  PwOut* oc_s = reinterpret_cast<PwOut*>(ch_s + CI_T);                    // [Cout4]
  float* w_s = reinterpret_cast<float*>(oc_s + Cout4);                    // [Cout4][CI_T]
  float* red_s = w_s + Cout4 * CI_T;                                      // [4][2*CI_T]
  float* st_s = red_s + 4 * 2 * CI_T;                                     // [4 warps][2*CI_T][32 lanes] running sums
  const int tid = threadIdx.x;
  // RING: [PW_RING_S] stages behind the statistics (16-byte aligned: every carve-up above is a multiple of 16 bytes)
  const uint32_t ring = smem_addr(st_s + 4 * 2 * CI_T * 32) + tid * 16;
  const int ci_base = blockIdx.y * CI_T;
  const int L = op.L_out, LQ = L >> 2;

  for (int col = tid; col < CI_T; col += PW_NT) {
    const int ci = ci_base + col;
    PwChan c = make_chan(op, ci < Cin ? ci : 0, true);
    if (ci >= Cin) c.g = nullptr;
    ch_s[col] = c;
  }
  for (int co = tid; co < Cout4; co += PW_NT) {
    PwOut o = {0.f, 0.f, 0.f};
    if (co < Cout) {
      const OutGradCoef k = out_grad_coef(op, co);
      o.A = k.A;
      o.Bx = k.Bx;
      o.Cc = k.Cc;
    }
    oc_s[co] = o;
  }
  for (int idx = tid; idx < Cout4 * CI_T; idx += PW_NT) {
    const int co = idx / CI_T, col = idx - co * CI_T;
    const int ci = ci_base + col;
    w_s[idx] = (co < Cout && ci < Cin) ? op.W[(size_t)co * Cin + ci] : 0.f;
  }
  __syncthreads();

  const uint64_t seed = load_seed(op.step_seed);
  const long long NQ = (long long)op.N * LQ;
  const bool has_bn = (op.out.bn >= 0 && op.out.g != nullptr);
  const bool need_x = has_bn || op.out_act == SEIST_OUT_SIGMOID;
  // BN-backward sums of the targets live in shared memory (one private slot per thread and statistic)
  // between quads: keeping them in registers costs 2*CI_T registers across the whole contraction loop
  float* my_st = st_s + (tid >> 5) * (2 * CI_T * 32) + (tid & 31);
#pragma unroll
  for (int i = 0; i < 2 * CI_T; ++i) my_st[i * 32] = 0.f;

  // RING: issue cursor over the flattened (quad group g, channel step) sequence, PW_RING_S - 1 steps ahead of the
  // consumer, so the copies of the next quad group are already in flight during the epilogue of the current one
  int ig = 0, ico = 0, istage = 0, cstage = 0;
  size_t iobase = 0;
  auto quad_base = [&](int g) -> size_t {
    const long long f = ((long long)blockIdx.x * G + g) * PW_NT + tid;
    const bool ok = f < NQ;
    const int n = ok ? (int)(f / LQ) : 0;
    const int l = ok ? (int)(f - (long long)n * LQ) * 4 : 0;
    return ((size_t)n * op.out.Ct + op.out.c0) * (size_t)L + l;
  };
  auto issue_step = [&]() {
    if (ig < G) {
      const uint32_t dst0 = ring + istage * PW_RING_STAGE_B;
#pragma unroll
      for (int j = 0; j < PW_BD_CG; ++j) {
        const size_t off = iobase + (size_t)min(ico + j, Cout - 1) * L;
        const uint32_t dst = dst0 + j * (3 * PW_NT * 16);
        if (op.out_dxd) cp_async16(dst, op.out_dxd + off);
        if (has_bn) cp_async16(dst + PW_NT * 16, op.out.g + off);
        if (need_x) cp_async16(dst + 2 * PW_NT * 16, op.out.x + off);
      }
      ico += PW_BD_CG;
      if (ico >= Cout4) {
        ico = 0;
        if (++ig < G) iobase = quad_base(ig);
      }
    }
    cp_async_commit();   // one group per step (possibly empty) keeps the wait count uniform
    istage = istage + 1 == PW_RING_S ? 0 : istage + 1;
  };
  if constexpr (RING) {
    iobase = quad_base(0);
#pragma unroll
    for (int s = 0; s < PW_RING_S - 1; ++s) issue_step();
  }

  for (int g = 0; g < G; ++g) {
    const long long f = ((long long)blockIdx.x * G + g) * PW_NT + tid;
    const bool ok = f < NQ;
    const int n = ok ? (int)(f / LQ) : 0;
    const int l = ok ? (int)(f - (long long)n * LQ) * 4 : 0;
    const float pf = path_factor(op, seed, n) * alpha_factor(op, seed, n);
    float2 acc[CI_T / 2][4];   // [target-channel pair][sample] (fma2 lanes = even / odd channel)
#pragma unroll
    for (int c = 0; c < CI_T / 2; ++c)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[c][q] = make_float2(0.f, 0.f);
    const size_t obase = ((size_t)n * op.out.Ct + op.out.c0) * (size_t)L + l;
    for (int co0 = 0; co0 < Cout4; co0 += PW_BD_CG) {
      float4 dx[PW_BD_CG], du[PW_BD_CG], xo[PW_BD_CG];
      if constexpr (RING) {
        issue_step();
        cp_async_wait<PW_RING_S - 1>();
        const uint32_t src0 = ring + cstage * PW_RING_STAGE_B;
        cstage = cstage + 1 == PW_RING_S ? 0 : cstage + 1;
#pragma unroll
        for (int j = 0; j < PW_BD_CG; ++j) {
          const uint32_t src = src0 + j * (3 * PW_NT * 16);
          dx[j] = op.out_dxd ? lds4(src) : make_float4(0.f, 0.f, 0.f, 0.f);
          du[j] = has_bn ? lds4(src + PW_NT * 16) : make_float4(0.f, 0.f, 0.f, 0.f);
          xo[j] = need_x ? lds4(src + 2 * PW_NT * 16) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      } else {
#pragma unroll
        for (int j = 0; j < PW_BD_CG; ++j) {
          const int co = min(co0 + j, Cout - 1);
          const size_t off = obase + (size_t)co * L;
          dx[j] = op.out_dxd ? ldg4(op.out_dxd + off) : make_float4(0.f, 0.f, 0.f, 0.f);
          du[j] = has_bn ? ldg4(op.out.g + off) : make_float4(0.f, 0.f, 0.f, 0.f);
          xo[j] = need_x ? ldg4(op.out.x + off) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
#pragma unroll
      for (int j = 0; j < PW_BD_CG; ++j) {
        const int co = co0 + j;
        const PwOut o = oc_s[co];
        float4 gv;
        gv.x = dx[j].x + fmaf(o.A, du[j].x, fmaf(o.Bx, xo[j].x, o.Cc));
        gv.y = dx[j].y + fmaf(o.A, du[j].y, fmaf(o.Bx, xo[j].y, o.Cc));
        gv.z = dx[j].z + fmaf(o.A, du[j].z, fmaf(o.Bx, xo[j].z, o.Cc));
        gv.w = dx[j].w + fmaf(o.A, du[j].w, fmaf(o.Bx, xo[j].w, o.Cc));
        if (op.out_act == SEIST_OUT_SIGMOID) {
          gv.x *= xo[j].x * (1.f - xo[j].x);
          gv.y *= xo[j].y * (1.f - xo[j].y);
          gv.z *= xo[j].z * (1.f - xo[j].z);
          gv.w *= xo[j].w * (1.f - xo[j].w);
        }
        gv.x *= pf;
        gv.y *= pf;
        gv.z *= pf;
        gv.w *= pf;
        if (F_ELEM) {
          const float4 kp = pw_keep4(op.p_elem, seed, op.seed_elem, ((uint64_t)n * Cout + min(co, Cout - 1)) * (uint64_t)L + l);
          gv.x *= kp.x;
          gv.y *= kp.y;
          gv.z *= kp.z;
          gv.w *= kp.w;
        }
        const float2* wr = reinterpret_cast<const float2*>(w_s + co * CI_T);   // zero rows for co >= Cout
        const float2 gx = dup2(gv.x), gy = dup2(gv.y), gz = dup2(gv.z), gw = dup2(gv.w);
#pragma unroll
        for (int cp = 0; cp < CI_T / 2; ++cp) {
          const float2 w = wr[cp];
          acc[cp][0] = fma2(w, gx, acc[cp][0]);
          acc[cp][1] = fma2(w, gy, acc[cp][1]);
          acc[cp][2] = fma2(w, gz, acc[cp][2]);
          acc[cp][3] = fma2(w, gw, acc[cp][3]);
        }
      }
    }
    if (!ok) continue;
    if constexpr (F_POOL) {
#pragma unroll
      for (int col = 0; col < CI_T; ++col) {
        const PwChan& c = ch_s[col];
        if (c.g == nullptr) continue;
        const float2(&ap)[4] = acc[col >> 1];
        float4 gg = (col & 1) ? make_float4(ap[0].y, ap[1].y, ap[2].y, ap[3].y) : make_float4(ap[0].x, ap[1].x, ap[2].x, ap[3].x);
        {
          // route the 4 pooled gradients to their 4*P source samples: g * (1/P + [first arg max])
          const long long soff = (long long)n * c.nstride + (long long)l * op.pool;
          float s1 = 0.f, s2 = 0.f;
          if (op.pool == 2) pool_route<2>(c, soff, gg, s1, s2);
          else if (op.pool == 4) pool_route<4>(c, soff, gg, s1, s2);
          else pool_route<8>(c, soff, gg, s1, s2);
          if (c.bn >= 0) {
            my_st[(2 * col) * 32] += s1;
            my_st[(2 * col + 1) * 32] += s2;
          }
        }
      }
    } else {
    // targets in batches of PW_BD_EB channels: all loads of a batch (x for khat / GELU', the old gradient when
    // accumulating) are issued before its first store, so their latency overlaps instead of serialising
    // load -> use -> store once per channel (the compiler cannot hoist loads over possibly aliasing stores)
#pragma unroll
    for (int cb = 0; cb < CI_T; cb += PW_BD_EB) {
      float4 xv[PW_BD_EB], ov[PW_BD_EB];
#pragma unroll
      for (int u = 0; u < PW_BD_EB; ++u) {
        const PwChan& c = ch_s[cb + u];
        const long long off = (long long)n * c.nstride + l;
        const bool live = c.g != nullptr;
        const bool want_x = live && ((F_GELU && c.act == SEIST_ACT_GELU) || c.bn >= 0);
        xv[u] = want_x ? ldg4(c.x + off) : make_float4(0.f, 0.f, 0.f, 0.f);
        ov[u] = (live && c.accum) ? ld4(c.g + off) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < PW_BD_EB; ++u) {
        const int col = cb + u;
        const PwChan& c = ch_s[col];
        if (c.g == nullptr) continue;
        const float2(&ap)[4] = acc[col >> 1];
        float4 gg = (col & 1) ? make_float4(ap[0].y, ap[1].y, ap[2].y, ap[3].y) : make_float4(ap[0].x, ap[1].x, ap[2].x, ap[3].x);
        const float4 x = xv[u];
        if (F_GELU && c.act == SEIST_ACT_GELU) {
          const float4 d = pw_gelu_grad4(make_float4(fmaf(c.sc, x.x, c.sh), fmaf(c.sc, x.y, c.sh), fmaf(c.sc, x.z, c.sh),
                                                     fmaf(c.sc, x.w, c.sh)));
          gg.x *= d.x;
          gg.y *= d.y;
          gg.z *= d.z;
          gg.w *= d.w;
        }
        if (c.bn >= 0) {
          my_st[(2 * col) * 32] += (gg.x + gg.y) + (gg.z + gg.w);
          my_st[(2 * col + 1) * 32] += fmaf(gg.x, (x.x - c.mu) * c.istd, gg.y * ((x.y - c.mu) * c.istd)) +
                                       fmaf(gg.z, (x.z - c.mu) * c.istd, gg.w * ((x.w - c.mu) * c.istd));
        }
        gg.x += ov[u].x;
        gg.y += ov[u].y;
        gg.z += ov[u].z;
        gg.w += ov[u].w;
        st4(c.g + (long long)n * c.nstride + l, gg);
      }
    }
    }
  }
  float st[2 * CI_T];
#pragma unroll
  for (int i = 0; i < 2 * CI_T; ++i) st[i] = my_st[i * 32];
  cta_reduce_atomic<2 * CI_T>(st, red_s, [&](int i, float s) {
    const PwChan& c = ch_s[i >> 1];
    if (c.g != nullptr && c.bn >= 0) {
      const SeistBN& e = op.bn_table[c.bn];
      atomicAdd(&e.gstat_acc[(i & 1) * e.C + c.bnc], (double)s);
    }
  });
}

// ================================================================================================
// backward (data), staged: one CTA owns a tile of 128 samples and ALL target channels of the op, so every output-channel
// operand (dxd | du | x) is read from memory once and its gradient combine (BN-backward, sigmoid', drop factors, dropout
// mask) is evaluated once, instead of once per 16-target tile.  Warp w holds targets 16w .. 16w+15 (same 16 x 4 register
// tile as pw_bwd_data_kernel, lane = quad of 4 samples).  The operands of PWS_CC output channels form one stage of a
// PWS_S-deep shared-memory ring filled with cp.async; the thread that copied a (channel, quad) slot combines it in place
// after its own wait_group, then one barrier publishes the stage to every warp.  Persistent grid over sample tiles.
// blockDim = 32 * ceil(Cin / 16).
// ================================================================================================
constexpr int PWS_CC = 8;                          // output channels per ring stage
constexpr int PWS_S = 3;                           // ring stages (PWS_S - 1 stages in flight while one is consumed)
constexpr int PWS_PLANE_B = 32 * 16;               // one channel plane of a tile: 32 quads x 16 bytes
constexpr int PWS_STAGE_B = PWS_CC * 3 * PWS_PLANE_B;   // [channel][dxd | du | x][quad] float4
constexpr int PWS_MAX_CIN = 192;                   // 12 warps

__device__ __forceinline__ void sts4(uint32_t a, float4 v) {
  asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// one reduce-scatter step: lanes with bit H set keep values [H, 2H), the others [0, H); each adds its partner's half
template <int H>
__device__ __forceinline__ void warp_halve(float* v, int lane) {
  const bool up = (lane & H) != 0;
#pragma unroll
  for (int k = 0; k < H; ++k) {
    const float send = up ? v[k] : v[k + H];
    const float keep = up ? v[k + H] : v[k];
    v[k] = keep + __shfl_xor_sync(0xffffffffu, send, H);
  }
}

template <bool F_ELEM, bool F_GELU>
__global__ void __launch_bounds__(PWS_MAX_CIN * 2) pw_bwd_data_staged_kernel(const __grid_constant__ SeistOp op) {
  extern __shared__ __align__(16) unsigned char sm_raw[];
  const int NT = blockDim.x, NW = NT >> 5;
  const int Cout = op.Cout, Cin = op.Cin, Cin16 = NW * 16;
  const int nck = (Cout + PWS_CC - 1) / PWS_CC, CoutC = nck * PWS_CC;
  PwChan* ch_s = reinterpret_cast<PwChan*>(sm_raw);                       // [Cin16] targets
  PwOut* oc_s = reinterpret_cast<PwOut*>(ch_s + Cin16);                   // [CoutC]
  float* w_s = reinterpret_cast<float*>(oc_s + CoutC);                    // [CoutC][Cin16]
  const uint32_t ring = smem_addr(w_s + CoutC * Cin16);                   // [PWS_S] stages (16-byte aligned carve-up)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int L = op.L_out, LQ = L >> 2;

  for (int ci = tid; ci < Cin16; ci += NT) {
    PwChan c = make_chan(op, ci < Cin ? ci : 0, true);
    if (ci >= Cin) c.g = nullptr;
    ch_s[ci] = c;
  }
  for (int co = tid; co < CoutC; co += NT) {
    PwOut o = {0.f, 0.f, 0.f};
    if (co < Cout) {
      const OutGradCoef k = out_grad_coef(op, co);
      o.A = k.A;
      o.Bx = k.Bx;
      o.Cc = k.Cc;
    }
    oc_s[co] = o;
  }
  for (int idx = tid; idx < CoutC * Cin16; idx += NT) {
    const int co = idx / Cin16, ci = idx - co * Cin16;
    w_s[idx] = (co < Cout && ci < Cin) ? op.W[(size_t)co * Cin + ci] : 0.f;
  }
  __syncthreads();

  const uint64_t seed = load_seed(op.step_seed);
  const long long NQ = (long long)op.N * LQ;
  const long long ntiles = (NQ + 31) / 32;
  const bool has_dxd = op.out_dxd != nullptr;
  const bool has_bn = (op.out.bn >= 0 && op.out.g != nullptr);
  const bool need_x = has_bn || op.out_act == SEIST_OUT_SIGMOID;
  auto quad_of = [&](long long tile, int& n, int& l) -> bool {
    const long long f = tile * 32 + lane;
    const bool ok = f < NQ;
    n = ok ? (int)(f / LQ) : 0;
    l = ok ? (int)(f - (long long)n * LQ) * 4 : 0;
    return ok;
  };

  // issue cursor over the flattened (tile, channel chunk) sequence, PWS_S - 1 stages ahead of the consumer; a thread
  // copies channels warp, warp + NW, ... of a chunk at quad `lane` (and later combines exactly those slots)
  long long itile = blockIdx.x;
  int ick = 0, istage = 0;
  int in_, il;
  bool iok = quad_of(itile, in_, il);
  size_t iobase = ((size_t)in_ * op.out.Ct + op.out.c0) * (size_t)L + il;
  auto issue_step = [&]() {
    if (itile < ntiles) {
      const uint32_t dst0 = ring + istage * PWS_STAGE_B + lane * 16;
      for (int c = warp; c < PWS_CC; c += NW) {
        const int co = ick * PWS_CC + c;
        if (iok && co < Cout) {
          const size_t off = iobase + (size_t)co * L;
          const uint32_t dst = dst0 + c * (3 * PWS_PLANE_B);
          if (has_dxd) cp_async16(dst, op.out_dxd + off);
          if (has_bn) cp_async16(dst + PWS_PLANE_B, op.out.g + off);
          if (need_x) cp_async16(dst + 2 * PWS_PLANE_B, op.out.x + off);
        }
      }
      if (++ick == nck) {
        ick = 0;
        itile += gridDim.x;
        iok = quad_of(itile, in_, il);
        iobase = ((size_t)in_ * op.out.Ct + op.out.c0) * (size_t)L + il;
      }
    }
    cp_async_commit();   // one group per step (possibly empty) keeps the wait count uniform
    istage = istage + 1 == PWS_S ? 0 : istage + 1;
  };
#pragma unroll
  for (int s = 0; s < PWS_S - 1; ++s) issue_step();

  bool warp_bn = false;   // any BN-backward target in this warp (warp-uniform)
  for (int t = 0; t < 16; ++t) {
    const PwChan& c = ch_s[warp * 16 + t];
    warp_bn |= c.g != nullptr && c.bn >= 0;
  }
  const PwChan* my_ch = ch_s + warp * 16;
  float st_run = 0.f;   // lane i: BN-backward sum (i & 1) of target warp * 16 + (i >> 1), over this CTA's tiles
  int cstage = 0;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    int n, l;
    const bool ok = quad_of(tile, n, l);
    const float pf = path_factor(op, seed, n) * alpha_factor(op, seed, n);
    float2 acc[8][4];   // [target pair][sample] (fma2 lanes = even / odd target)
#pragma unroll
    for (int c = 0; c < 8; ++c)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[c][q] = make_float2(0.f, 0.f);
    for (int ck = 0; ck < nck; ++ck) {
      cp_async_wait<PWS_S - 2>();
      const uint32_t st = ring + cstage * PWS_STAGE_B + lane * 16;
      cstage = cstage + 1 == PWS_S ? 0 : cstage + 1;
      for (int c = warp; c < PWS_CC; c += NW) {
        const int co = ck * PWS_CC + c;
        const uint32_t slot = st + c * (3 * PWS_PLANE_B);
        float4 gv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ok && co < Cout) {
          const float4 dx = has_dxd ? lds4(slot) : make_float4(0.f, 0.f, 0.f, 0.f);
          const float4 du = has_bn ? lds4(slot + PWS_PLANE_B) : make_float4(0.f, 0.f, 0.f, 0.f);
          const float4 xo = need_x ? lds4(slot + 2 * PWS_PLANE_B) : make_float4(0.f, 0.f, 0.f, 0.f);
          const PwOut o = oc_s[co];
          gv.x = dx.x + fmaf(o.A, du.x, fmaf(o.Bx, xo.x, o.Cc));
          gv.y = dx.y + fmaf(o.A, du.y, fmaf(o.Bx, xo.y, o.Cc));
          gv.z = dx.z + fmaf(o.A, du.z, fmaf(o.Bx, xo.z, o.Cc));
          gv.w = dx.w + fmaf(o.A, du.w, fmaf(o.Bx, xo.w, o.Cc));
          if (op.out_act == SEIST_OUT_SIGMOID) {
            gv.x *= xo.x * (1.f - xo.x);
            gv.y *= xo.y * (1.f - xo.y);
            gv.z *= xo.z * (1.f - xo.z);
            gv.w *= xo.w * (1.f - xo.w);
          }
          gv.x *= pf;
          gv.y *= pf;
          gv.z *= pf;
          gv.w *= pf;
          if (F_ELEM) {
            const float4 kp = pw_keep4(op.p_elem, seed, op.seed_elem, ((uint64_t)n * Cout + co) * (uint64_t)L + l);
            gv.x *= kp.x;
            gv.y *= kp.y;
            gv.z *= kp.z;
            gv.w *= kp.w;
          }
        }
        sts4(slot, gv);   // channels past Cout / quads past the end contribute zeros
      }
      __syncthreads();
      issue_step();       // refills the slot every warp finished reading before the barrier
      const float* wr0 = w_s + ck * PWS_CC * Cin16 + warp * 16;
#pragma unroll
      for (int c = 0; c < PWS_CC; ++c) {
        const float4 g = lds4(st + c * (3 * PWS_PLANE_B));
        const float2* wr = reinterpret_cast<const float2*>(wr0 + c * Cin16);
        const float2 gx = dup2(g.x), gy = dup2(g.y), gz = dup2(g.z), gw = dup2(g.w);
#pragma unroll
        for (int cp = 0; cp < 8; ++cp) {
          const float2 w = wr[cp];
          acc[cp][0] = fma2(w, gx, acc[cp][0]);
          acc[cp][1] = fma2(w, gy, acc[cp][1]);
          acc[cp][2] = fma2(w, gz, acc[cp][2]);
          acc[cp][3] = fma2(w, gw, acc[cp][3]);
        }
      }
    }
    // epilogue of this warp's targets, in batches of PW_BD_EB channels (all loads of a batch before its first store)
    float bs[32];   // [2 * target + k]: BN-backward sums of this quad
#pragma unroll
    for (int cb = 0; cb < 16; cb += PW_BD_EB) {
      float4 xv[PW_BD_EB], ov[PW_BD_EB];
#pragma unroll
      for (int u = 0; u < PW_BD_EB; ++u) {
        const PwChan& c = my_ch[cb + u];
        const long long off = (long long)n * c.nstride + l;
        const bool live = ok && c.g != nullptr;
        const bool want_x = live && ((F_GELU && c.act == SEIST_ACT_GELU) || c.bn >= 0);
        xv[u] = want_x ? ldg4(c.x + off) : make_float4(0.f, 0.f, 0.f, 0.f);
        ov[u] = (live && c.accum) ? ld4(c.g + off) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < PW_BD_EB; ++u) {
        const int col = cb + u;
        const PwChan& c = my_ch[col];
        bs[2 * col] = 0.f;
        bs[2 * col + 1] = 0.f;
        if (!ok || c.g == nullptr) continue;
        const float2(&ap)[4] = acc[col >> 1];
        float4 gg = (col & 1) ? make_float4(ap[0].y, ap[1].y, ap[2].y, ap[3].y) : make_float4(ap[0].x, ap[1].x, ap[2].x, ap[3].x);
        const float4 x = xv[u];
        if (F_GELU && c.act == SEIST_ACT_GELU) {
          const float4 d = pw_gelu_grad4(make_float4(fmaf(c.sc, x.x, c.sh), fmaf(c.sc, x.y, c.sh), fmaf(c.sc, x.z, c.sh),
                                                     fmaf(c.sc, x.w, c.sh)));
          gg.x *= d.x;
          gg.y *= d.y;
          gg.z *= d.z;
          gg.w *= d.w;
        }
        if (c.bn >= 0) {
          bs[2 * col] = (gg.x + gg.y) + (gg.z + gg.w);
          bs[2 * col + 1] = fmaf(gg.x, (x.x - c.mu) * c.istd, gg.y * ((x.y - c.mu) * c.istd)) +
                            fmaf(gg.z, (x.z - c.mu) * c.istd, gg.w * ((x.w - c.mu) * c.istd));
        }
        gg.x += ov[u].x;
        gg.y += ov[u].y;
        gg.z += ov[u].z;
        gg.w += ov[u].w;
        st4(c.g + (long long)n * c.nstride + l, gg);
      }
    }
    if (warp_bn) {
      // reduce-scatter over the warp (31 shuffles): afterwards bs[0] of lane i is the warp's sum of value i
      warp_halve<16>(bs, lane);
      warp_halve<8>(bs, lane);
      warp_halve<4>(bs, lane);
      warp_halve<2>(bs, lane);
      warp_halve<1>(bs, lane);
      st_run += bs[0];
    }
  }
  cp_async_wait<0>();
  if (warp_bn) {
    const PwChan& c = my_ch[lane >> 1];
    if (c.g != nullptr && c.bn >= 0) {
      const SeistBN& e = op.bn_table[c.bn];
      atomicAdd(&e.gstat_acc[(lane & 1) * e.C + c.bnc], (double)st_run);
    }
  }
}

// ================================================================================================
// backward: residual pass-through, vectorised.  grid (ceil(NQ/(128*G)), Cout): one channel per CTA.
// ================================================================================================
__global__ void __launch_bounds__(PW_NT) res_bwd4_kernel(const __grid_constant__ SeistOp op, const int G) {
  __shared__ float red_s[4 * 4];
  const int tid = threadIdx.x;
  const int co = blockIdx.y;
  const int L = op.L_out, LQ = L >> 2;
  const long long NQ = (long long)op.N * LQ;
  const uint64_t seed = load_seed(op.step_seed);
  const OutGradCoef kc = out_grad_coef(op, co);
  const bool has_bn = (op.out.bn >= 0 && op.out.g != nullptr);
  const bool need_x = has_bn || op.out_act == SEIST_OUT_SIGMOID;
  const SeistView& va = op.res_a;
  const SeistView& vb = op.res_b;
  const bool wa = va.C > 0 && va.g != nullptr, wb = vb.C > 0 && vb.g != nullptr;
  float amu = 0.f, aistd = 0.f, bmu = 0.f, bistd = 0.f;
  if (wa && va.bn >= 0) view_khat(op, va, co, amu, aistd);
  if (wb && vb.bn >= 0) view_khat(op, vb, co, bmu, bistd);
  float st[4] = {0.f, 0.f, 0.f, 0.f};
  for (int g = 0; g < G; ++g) {
    const long long f = ((long long)blockIdx.x * G + g) * PW_NT + tid;
    if (f >= NQ) break;
    const int n = (int)(f / LQ);
    const int l = (int)(f - (long long)n * LQ) * 4;
    const size_t off = ((size_t)n * op.out.Ct + op.out.c0 + co) * (size_t)L + l;
    float4 gv = op.out_dxd ? ldg4(op.out_dxd + off) : make_float4(0.f, 0.f, 0.f, 0.f);
    if (need_x) {
      const float4 x = ldg4(op.out.x + off);
      if (has_bn) {
        const float4 du = ldg4(op.out.g + off);
        gv.x += fmaf(kc.A, du.x, fmaf(kc.Bx, x.x, kc.Cc));
        gv.y += fmaf(kc.A, du.y, fmaf(kc.Bx, x.y, kc.Cc));
        gv.z += fmaf(kc.A, du.z, fmaf(kc.Bx, x.z, kc.Cc));
        gv.w += fmaf(kc.A, du.w, fmaf(kc.Bx, x.w, kc.Cc));
      }
      if (op.out_act == SEIST_OUT_SIGMOID) {
        gv.x *= x.x * (1.f - x.x);
        gv.y *= x.y * (1.f - x.y);
        gv.z *= x.z * (1.f - x.z);
        gv.w *= x.w * (1.f - x.w);
      }
    }
#pragma unroll
    for (int which = 0; which < 2; ++which) {
      const SeistView& v = which == 0 ? va : vb;
      if (!(which == 0 ? wa : wb)) continue;
      float4 gg = gv;
      if (which == 0) {
        const float af = alpha_factor(op, seed, n);
        gg.x *= af;
        gg.y *= af;
        gg.z *= af;
        gg.w *= af;
      }
      const size_t voff = ((size_t)n * v.Ct + v.c0 + co) * (size_t)L + l;
      if (v.bn >= 0) {
        const float4 x = ldg4(v.x + voff);
        const float mu = which == 0 ? amu : bmu, is = which == 0 ? aistd : bistd;
        st[2 * which] += (gg.x + gg.y) + (gg.z + gg.w);
        st[2 * which + 1] += fmaf(gg.x, (x.x - mu) * is, gg.y * ((x.y - mu) * is)) +
                             fmaf(gg.z, (x.z - mu) * is, gg.w * ((x.w - mu) * is));
      }
      float* gp = v.g + voff;
      if (v.accum) {
        const float4 old = ld4(gp);
        gg.x += old.x;
        gg.y += old.y;
        gg.z += old.z;
        gg.w += old.w;
      }
      st4(gp, gg);
    }
  }
  cta_reduce_atomic<4>(st, red_s, [&](int i, float s) {
    const SeistView& v = (i >> 1) == 0 ? va : vb;
    const bool w = (i >> 1) == 0 ? wa : wb;
    if (w && v.bn >= 0) {
      const SeistBN& e = op.bn_table[v.bn];
      atomicAdd(&e.gstat_acc[(i & 1) * e.C + v.bn_c0 + co], (double)s);
    }
  });
}

// ================================================================================================
// launchers
// ================================================================================================
// pooled input (AvgPool + MaxPool in front of the 1x1 conv): one un-activated view of exactly pool * L_out
// samples, no dropout / residual in the epilogue (true for every LAAB / KV-aggregation conv of the family)
static bool pw_pooled_ok(const SeistOp& op) {
  if (op.pool != 2 && op.pool != 4 && op.pool != 8) return false;
  if (op.n_in != 1 || op.in[0].act != SEIST_ACT_NONE || op.in[0].L != op.L_out * op.pool) return false;
  return op.p_elem <= 0.f && op.res_a.C == 0 && op.res_b.C == 0;
}
bool pw_eligible(const SeistOp& op) {
  if (op.k != 1 || op.stride != 1 || op.groups != 1 || op.up_src_L > 0) return false;
  if (op.L_out & 3) return false;
  if (op.pool > 1) return pw_pooled_ok(op);
  return true;
}

static int pick_G(long long nq, int tiles_y, int sm_count) {
  // enough CTAs for ~4 waves, but several quads per thread (at most 8) to amortise the per-CTA setup / reduction
  long long ctas = (nq + PW_NT - 1) / PW_NT;
  int G = 1;
  while (G < 8 && (ctas / (2 * G)) * tiles_y >= 4LL * sm_count) G *= 2;
  return G;
}

template <typename K>
static int pw_set_smem(K kernel, size_t bytes) {
  if (bytes > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return (int)e;
  }
  return 0;
}

static bool any_gelu(const SeistOp& op) {
  for (int i = 0; i < op.n_in; ++i)
    if (op.in[i].act == SEIST_ACT_GELU) return true;
  return false;
}

template <int COT, bool E, bool R, bool Gf, bool P = false>
static int pw_fwd_go(const SeistOp& op, cudaStream_t s, dim3 grid, size_t smem, int G) {
  int rc = pw_set_smem(pw_fwd_kernel<COT, E, R, Gf, P>, smem);
  if (!rc) pw_fwd_kernel<COT, E, R, Gf, P><<<grid, PW_NT, smem, s>>>(op, G);
  return rc;
}
template <int COT>
static int pw_fwd_sel(const SeistOp& op, cudaStream_t s, dim3 grid, size_t smem, int G) {
  if (op.pool > 1) return pw_fwd_go<COT, false, false, false, true>(op, s, grid, smem, G);
  const int sel = (op.p_elem > 0.f ? 4 : 0) | ((op.res_a.C > 0 || op.res_b.C > 0) ? 2 : 0) | (any_gelu(op) ? 1 : 0);
  switch (sel) {
    case 0: return pw_fwd_go<COT, false, false, false>(op, s, grid, smem, G);
    case 1: return pw_fwd_go<COT, false, false, true>(op, s, grid, smem, G);
    case 2: return pw_fwd_go<COT, false, true, false>(op, s, grid, smem, G);
    case 3: return pw_fwd_go<COT, false, true, true>(op, s, grid, smem, G);
    case 4: return pw_fwd_go<COT, true, false, false>(op, s, grid, smem, G);
    case 5: return pw_fwd_go<COT, true, false, true>(op, s, grid, smem, G);
    case 6: return pw_fwd_go<COT, true, true, false>(op, s, grid, smem, G);
    default: return pw_fwd_go<COT, true, true, true>(op, s, grid, smem, G);
  }
}

int launch_pw_fwd(const SeistOp& op, cudaStream_t s, int sm_count) {
  const int cot = op.Cout > 8 ? 16 : 8;
  const int Cin8 = (op.Cin + 7) & ~7;
  const size_t smem = sizeof(PwChan) * Cin8 + sizeof(float) * ((size_t)Cin8 * cot + 5 * cot + 4 * 2 * cot + 4 * 2 * cot * 32);
  const long long nq = (long long)op.N * (op.L_out >> 2);
  const int ty = (op.Cout + cot - 1) / cot;
  const int G = pick_G(nq, ty, sm_count);
  dim3 grid((unsigned)((nq + (long long)PW_NT * G - 1) / ((long long)PW_NT * G)), ty);
  const int rc = cot == 16 ? pw_fwd_sel<16>(op, s, grid, smem, G) : pw_fwd_sel<8>(op, s, grid, smem, G);
  if (rc) return rc;
  note_launch();
  return check_launch("pw_fwd");
}

template <int CIT, bool E, bool Gf, bool P = false>
static int pw_bwdd_go(const SeistOp& op, cudaStream_t s, dim3 grid, size_t smem, int G) {
  if (!P) smem += (size_t)PW_RING_S * PW_RING_STAGE_B;   // operand ring
  int rc = pw_set_smem(pw_bwd_data_kernel<CIT, E, Gf, P>, smem);
  if (!rc) pw_bwd_data_kernel<CIT, E, Gf, P><<<grid, PW_NT, smem, s>>>(op, G);
  return rc;
}
template <int CIT>
static int pw_bwdd_sel(const SeistOp& op, cudaStream_t s, dim3 grid, size_t smem, int G) {
  if (op.pool > 1) return pw_bwdd_go<CIT, false, false, true>(op, s, grid, smem, G);
  const int sel = (op.p_elem > 0.f ? 2 : 0) | (any_gelu(op) ? 1 : 0);
  switch (sel) {
    case 0: return pw_bwdd_go<CIT, false, false>(op, s, grid, smem, G);
    case 1: return pw_bwdd_go<CIT, false, true>(op, s, grid, smem, G);
    case 2: return pw_bwdd_go<CIT, true, false>(op, s, grid, smem, G);
    default: return pw_bwdd_go<CIT, true, true>(op, s, grid, smem, G);
  }
}

int launch_pw_bwd_data(const SeistOp& op, cudaStream_t s, int sm_count) {
  const int cit = op.Cin > 8 ? 16 : 8;
  const int Cout4 = (op.Cout + 3) & ~3;
  const size_t smem = sizeof(PwChan) * cit + sizeof(PwOut) * Cout4 + sizeof(float) * ((size_t)Cout4 * cit + 4 * 2 * cit + 4 * 2 * cit * 32);
  const long long nq = (long long)op.N * (op.L_out >> 2);
  const int ty = (op.Cin + cit - 1) / cit;
  const int G = pick_G(nq, ty, sm_count);
  dim3 grid((unsigned)((nq + (long long)PW_NT * G - 1) / ((long long)PW_NT * G)), ty);
  const int rc = cit == 16 ? pw_bwdd_sel<16>(op, s, grid, smem, G) : pw_bwdd_sel<8>(op, s, grid, smem, G);
  if (rc) return rc;
  note_launch();
  return check_launch("pw_bwd_data");
}

static size_t pw_bwd_data_staged_smem(const SeistOp& op) {
  const int cin16 = (op.Cin + 15) & ~15, coutc = (op.Cout + PWS_CC - 1) / PWS_CC * PWS_CC;
  return sizeof(PwChan) * cin16 + sizeof(PwOut) * coutc + sizeof(float) * (size_t)coutc * cin16 + (size_t)PWS_S * PWS_STAGE_B;
}

// Non-pooled 1x1 data gradients with more than one 16-target tile, whose weights and ring fit one CTA's shared memory.
// Two-tile ops (Cin <= 32) with a GELU target stay on pw_bwd_data_kernel: there the staged CTA is two warps whose GELU'
// epilogue is not hidden behind the ring, and it measured slower on H100 than reading the operands twice.
bool pw_bwd_data_staged_ok(const SeistOp& op) {
  return pw_eligible(op) && op.pool <= 1 && op.Cin > 16 && op.Cin <= PWS_MAX_CIN && (op.Cin > 32 || !any_gelu(op)) &&
         pw_bwd_data_staged_smem(op) <= 227 * 1024;
}

template <bool E, bool Gf>
static int pw_bwdd_staged_go(const SeistOp& op, cudaStream_t s, int sm_count) {
  const auto kernel = pw_bwd_data_staged_kernel<E, Gf>;
  const size_t smem = pw_bwd_data_staged_smem(op);
  const int nt = 32 * ((op.Cin + 15) / 16);
  int rc = pw_set_smem(kernel, smem);
  if (rc) return rc;
  int per_sm = 0;
  const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, nt, smem);
  if (e != cudaSuccess) return (int)e;
  if (per_sm < 1) {
    set_error("pw_bwd_data_staged: no resident CTA fits");
    return -2;
  }
  const long long tiles = ((long long)op.N * (op.L_out >> 2) + 31) / 32;
  const long long resident = (long long)per_sm * sm_count;
  const long long grid = tiles < resident ? tiles : resident;
  kernel<<<(unsigned)grid, nt, smem, s>>>(op);
  return 0;
}

int launch_pw_bwd_data_staged(const SeistOp& op, cudaStream_t s, int sm_count) {
  const int sel = (op.p_elem > 0.f ? 2 : 0) | (any_gelu(op) ? 1 : 0);
  int rc;
  switch (sel) {
    case 0: rc = pw_bwdd_staged_go<false, false>(op, s, sm_count); break;
    case 1: rc = pw_bwdd_staged_go<false, true>(op, s, sm_count); break;
    case 2: rc = pw_bwdd_staged_go<true, false>(op, s, sm_count); break;
    default: rc = pw_bwdd_staged_go<true, true>(op, s, sm_count); break;
  }
  if (rc) return rc;
  note_launch();
  return check_launch("pw_bwd_data_staged");
}

int launch_res_bwd4(const SeistOp& op, cudaStream_t s, int sm_count) {
  const long long nq = (long long)op.N * (op.L_out >> 2);
  const int G = pick_G(nq, op.Cout, sm_count);
  dim3 grid((unsigned)((nq + (long long)PW_NT * G - 1) / ((long long)PW_NT * G)), op.Cout);
  res_bwd4_kernel<<<grid, PW_NT, 0, s>>>(op, G);
  note_launch();
  return check_launch("res_bwd4");
}

// ================================================================================================
// backward (weights), groups == 1, any k / stride / up-sampled input:
//   dW[co][r] = sum_{n,l} gacc[co][n,l] * convin[ci(r)][n, l*S + t(r) - pad_left],   r = ci*k + t
//
// A CTA owns a CO_B x R_B tile of dW and a strided share of all 128-sample chunks.  Per chunk every
// needed element is loaded (all loads of the chunk in flight at once), transformed ONCE (BN-backward
// prologue for gacc; BN-apply / GELU / up-sampling / padding for the input) and parked in shared
// memory; the threads then form TG = (CO_B/4)*(R_B/8) tile coordinates x PG sample groups: each thread
// keeps a 4 x 8 register tile and walks its sample quads (k = 1: 12 LDS.128 per 128 FMA).  Sample groups
// are folded through shared memory once at the end; one float atomic per dW element per CTA.
// ================================================================================================
constexpr int BW_NT = 256;

// BW_PC = output samples per chunk (128, or 512 for narrow tiles where the per-chunk barriers/latency dominate)
template <int CO_B, int R_B, bool K1, int BW_PC>
__global__ void __launch_bounds__(BW_NT, 3) bww_kernel(const __grid_constant__ SeistOp op, const int nci_max, const int g_async, const int gx_off) {
  constexpr int BW_PITCH = BW_PC + 4;   // input row pitch (floats), keeps 16-byte alignment
  constexpr int BW_GP = 2 * BW_PC + 8;  // gacc channel-PAIR row pitch: g_s[pr][2*s + half] (fma2 operand pairs)
  extern __shared__ __align__(16) unsigned char sm_raw[];
  constexpr int TGM = CO_B / 4, TGN = R_B / 8, TG = TGM * TGN, PG = BW_NT / TG;
  static_assert(TG <= BW_NT && BW_NT % TG == 0, "bad tile");
  const int k = op.k, S = op.stride, L = op.L_out;
  const int gs_in = op.Cin / op.groups, gs_out = op.Cout / op.groups;
  const int tpg = (gs_out + CO_B - 1) / CO_B;            // output-channel tiles per group
  const int grp = blockIdx.y / tpg;
  const int Cin = (grp + 1) * gs_in;                      // channel bounds of THIS group
  const int Cout = (grp + 1) * gs_out;
  const int R = gs_in * k;
  const int width = BW_PC * S + k - S;
  const int pitch = K1 ? BW_PITCH : (width | 1);            // odd pitch: scalar reads spread over banks
  const int stage_f = (CO_B / 2) * BW_GP + nci_max * pitch;
  const int area_f = stage_f > BW_NT * 36 ? stage_f : BW_NT * 36;
  float* g_s = reinterpret_cast<float*>(sm_raw);            // [CO_B/2][BW_GP]
  float* in_s = g_s + (CO_B / 2) * BW_GP;                   // [nci][pitch]
  PwOut* oc_s = reinterpret_cast<PwOut*>(g_s + ((area_f + 3) & ~3));   // [CO_B]
  PwChan* ch_s = reinterpret_cast<PwChan*>(oc_s + CO_B);                // [nci_max] (k = 1 fast path)
  float* src_s = reinterpret_cast<float*>(ch_s + nci_max + 1);          // [nci_max][width+4] (up-sampled input only)
  float* gx_s = reinterpret_cast<float*>(sm_raw) + gx_off;              // [2][CO_B/2][BW_GP] raw x / dxd planes (g_async)
  float* gd_s = gx_s + (CO_B / 2) * BW_GP;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int co_base = grp * gs_out + (blockIdx.y - grp * tpg) * CO_B, r_base = blockIdx.z * R_B;
  const int ci_lo = grp * gs_in + r_base / k;
  const int ci_hi = min(grp * gs_in + (r_base + R_B - 1) / k, Cin - 1);
  const int nci = ci_hi - ci_lo + 1;

  for (int col = tid; col < CO_B; col += BW_NT) {
    const int co = co_base + col;
    PwOut o = {0.f, 0.f, 0.f};
    if (co < Cout) {
      const OutGradCoef kc = out_grad_coef(op, co);
      o.A = kc.A;
      o.Bx = kc.Bx;
      o.Cc = kc.Cc;
    }
    oc_s[col] = o;
  }
  if (K1)
    for (int row = tid; row < nci; row += BW_NT) ch_s[row] = make_chan(op, ci_lo + row, false);
  __syncthreads();

  const uint64_t seed = load_seed(op.step_seed);
  const bool has_bn = (op.out.bn >= 0 && op.out.g != nullptr);
  const bool need_x = has_bn || op.out_act == SEIST_OUT_SIGMOID;
  const bool vec = (L & 3) == 0;
  const bool plain = op.pool <= 1 && op.up_src_L == 0;
  const int Lsrc = op.in[0].L;
  const float ratio = op.up_src_L > 0 ? (float)Lsrc / (float)op.L_in : 1.f;
  const int tcoord = tid % TG, pg = tid / TG;
  const int tm = tcoord / TGN, tn = tcoord % TGN;
  int roff[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int r = r_base + tn + TGN * j;          // interleaved columns: lanes of a warp read adjacent rows
    const int rr = r < R ? r : r_base;            // padded columns read valid memory; never written back
    const int q = rr / k, t = rr - q * k;               // q: input channel inside the group
    roff[j] = (grp * gs_in + q - ci_lo) * pitch + t;
  }
  float2 acc[2][8];   // [pair row ip][column]: channels 2*(tm + TGM*ip) + {0 (.x), 1 (.y)}
  float2 bacc[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = make_float2(0.f, 0.f);

  const int chunks_per_n = (L + BW_PC - 1) / BW_PC;
  const int total = op.N * chunks_per_n;
  constexpr int QPR = BW_PC / 4;
  for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
    const int n = tile / chunks_per_n;
    const int l0 = (tile - n * chunks_per_n) * BW_PC;
    const float pf = path_factor(op, seed, n) * alpha_factor(op, seed, n);
    // ---- conv-input rows, k = 1 fast path: raw 16-byte asynchronous copies, ALL in flight at once and behind the
    // gacc loads below; every thread later transforms its own quads in place (no barrier in between).  A
    // load -> transform -> store loop would expose one memory latency per quad
    const bool in_async = K1 && vec && plain;
    if (in_async) {
      for (int idx = tid; idx < nci * QPR; idx += BW_NT) {
        const int row = idx / QPR, q = idx - row * QPR;
        const int l = l0 + 4 * q;
        float* dst = in_s + row * pitch + 4 * q;
        if (l < L) {
          const PwChan& c = ch_s[row];
          cp_async16(smem_addr(dst), c.x + (long long)n * c.nstride + l);
        } else {
          st4(dst, make_float4(0.f, 0.f, 0.f, 0.f));
        }
      }
      cp_async_commit();
    }
    // ---- gacc rows ------------------------------------------------------------------------------
    if (vec && g_async) {
      gacc_issue<BW_NT>(op, n, l0, L, co_base, Cout, CO_B, QPR, BW_GP, g_s, gx_s, gd_s, has_bn, need_x);
      cp_async_commit();
      cp_async_wait<0>();
      gacc_combine<BW_NT>(op, n, l0, L, co_base, Cout, CO_B, QPR, BW_GP, g_s, gx_s, gd_s, oc_s, has_bn, need_x, pf, seed, op.Cout);
    } else if (vec) {
      for (int idx = tid; idx < (CO_B / 2) * QPR; idx += BW_NT) {
        const int pr = idx / QPR, q = idx - pr * QPR;
        const int l = l0 + 4 * q;
        float4 gh[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = 2 * pr + h, co = co_base + row;
          float4 gv = make_float4(0.f, 0.f, 0.f, 0.f);
          if (co < Cout && l < L) {
            const size_t off = ((size_t)n * op.out.Ct + op.out.c0 + co) * (size_t)L + l;
            if (op.out_dxd) gv = ldg4(op.out_dxd + off);
            if (need_x) {
              const float4 x = ldg4(op.out.x + off);
              if (has_bn) {
                const float4 du = ldg4(op.out.g + off);
                const PwOut o = oc_s[row];
                gv = add4(gv, fma4(splat4(o.A), du, fma4(splat4(o.Bx), x, splat4(o.Cc))));
              }
              if (op.out_act == SEIST_OUT_SIGMOID) gv = mul4(gv, mul4(x, fma4(x, splat4(-1.f), splat4(1.f))));
            }
            gv = scale4(gv, pf);
            if (op.p_elem > 0.f) gv = mul4(gv, keep4(op.p_elem, seed, op.seed_elem, ((uint64_t)n * Cout + co) * (uint64_t)L + l));
          }
          gh[h] = gv;
        }
        float* gp = g_s + pr * BW_GP + 8 * q;
        st4(gp, make_float4(gh[0].x, gh[1].x, gh[0].y, gh[1].y));
        st4(gp + 4, make_float4(gh[0].z, gh[1].z, gh[0].w, gh[1].w));
      }
    } else {
      for (int idx = tid; idx < CO_B * BW_PC; idx += BW_NT) {
        const int row = idx / BW_PC, pos = idx - row * BW_PC;
        const int co = co_base + row, l = l0 + pos;
        float v = 0.f;
        if (co < Cout && l < L) {
          OutGradCoef kc;
          kc.A = oc_s[row].A;
          kc.Bx = oc_s[row].Bx;
          kc.Cc = oc_s[row].Cc;
          v = out_grad_at(op, kc, n, co, l) * pf * elem_factor(op, seed, n, co, l);
        }
        g_s[(row >> 1) * BW_GP + 2 * pos + (row & 1)] = v;
      }
    }
    // ---- conv-input rows --------------------------------------------------------------------------
    const int p_base = l0 * S - op.pad_left;
    if (K1 && vec && op.pool > 1 && op.up_src_L == 0 && op.in[0].act == SEIST_ACT_NONE && Lsrc == L * op.pool &&
        (op.pool == 2 || op.pool == 4 || op.pool == 8)) {
      for (int idx = tid; idx < nci * QPR; idx += BW_NT) {
        const int row = idx / QPR, q = idx - row * QPR;
        const int l = l0 + 4 * q;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (l < L) {
          const PwChan& c = ch_s[row];
          v = pw_load_pooled(c.x + (long long)n * c.nstride + (long long)l * op.pool, op.pool, c.sc, c.sh);
        }
        st4(in_s + row * pitch + 4 * q, v);
      }
    } else if (in_async) {
      cp_async_wait<0>();
      for (int idx = tid; idx < nci * QPR; idx += BW_NT) {
        const int row = idx / QPR, q = idx - row * QPR;
        const PwChan& c = ch_s[row];
        if (l0 + 4 * q < L && (c.act != SEIST_ACT_NONE || c.sc != 1.f || c.sh != 0.f)) {
          float* dst = in_s + row * pitch + 4 * q;
          st4(dst, apply_view2(ld4(dst), c.sc, c.sh, c.act));
        }
      }
    } else {
      if (op.up_src_L > 0) {
        stage_upsampled_rows(op, n, ci_lo, nci, in_s, pitch, width, p_base, src_s, width + 4, Lsrc, ratio);
      } else
      if (plain) {
        rows_issue_plain(op, n, ci_lo, nci, nci, in_s, pitch, width, p_base);
        cp_async_commit();
        cp_async_wait<0>();
        rows_transform_plain(op, n, ci_lo, nci, in_s, pitch, width, p_base);
      } else {
        for (int r = warp; r < nci; r += BW_NT / 32) {
          const RowSrc rs = make_row(op, n, ci_lo + r);
          float* dst = in_s + r * pitch;
          for (int pos = lane; pos < width; pos += 32) dst[pos] = conv_input_at(op, rs, p_base + pos, Lsrc, ratio);
        }
      }
    }
    __syncthreads();
    // ---- accumulate ---------------------------------------------------------------------------------
    for (int q = pg; q < QPR; q += PG) {
      float2 gp[2][4];   // [pair row][sample]
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float* gr = g_s + (tm + TGM * i) * BW_GP + 8 * q;
        const float4 a = ld4(gr), b = ld4(gr + 4);
        gp[i][0] = make_float2(a.x, a.y);
        gp[i][1] = make_float2(a.z, a.w);
        gp[i][2] = make_float2(b.x, b.y);
        gp[i][3] = make_float2(b.z, b.w);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float4 iq;
        if (K1) {
          iq = ld4(in_s + roff[j] + 4 * q);
        } else {
          const float* ip = in_s + roff[j] + 4 * q * S;
          iq = make_float4(ip[0], ip[S], ip[2 * S], ip[3 * S]);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float2 a = acc[i][j];
          a = fma2(gp[i][0], dup2(iq.x), a);
          a = fma2(gp[i][1], dup2(iq.y), a);
          a = fma2(gp[i][2], dup2(iq.z), a);
          a = fma2(gp[i][3], dup2(iq.w), a);
          acc[i][j] = a;
        }
      }
      if (tn == 0) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          bacc[i].x += (gp[i][0].x + gp[i][1].x) + (gp[i][2].x + gp[i][3].x);
          bacc[i].y += (gp[i][0].y + gp[i][1].y) + (gp[i][2].y + gp[i][3].y);
        }
      }
    }
    __syncthreads();
  }

  // ---- fold the sample groups through shared memory (reuses the staging area) -------------------------
  float* red = g_s;
  constexpr int RW = 36;
  float* mine = red + (size_t)tid * RW;
#pragma unroll
  for (int i = 0; i < 4; ++i) {   // slot i <-> channel 2*(tm + TGM*(i>>1)) + (i&1)
#pragma unroll
    for (int j = 0; j < 8; ++j) mine[i * 8 + j] = (i & 1) ? acc[i >> 1][j].y : acc[i >> 1][j].x;
    mine[32 + i] = (i & 1) ? bacc[i >> 1].y : bacc[i >> 1].x;
  }
  __syncthreads();
  for (int idx = tid; idx < TG * RW; idx += BW_NT) {
    const int tc = idx / RW, e = idx - tc * RW;
    float s = 0.f;
    for (int p = 0; p < PG; ++p) s += red[((size_t)p * TG + tc) * RW + e];
    const int m = tc / TGN, nn = tc % TGN;
    if (e < 32) {
      const int i = e >> 3;
      const int co = co_base + 2 * (m + TGM * (i >> 1)) + (i & 1), r = r_base + nn + TGN * (e & 7);
      if (co < Cout && r < R) atomicAdd(&op.dW[(size_t)co * R + r], s);   // W is [Cout][gs_in][k]: row co, column r
    } else if (nn == 0 && blockIdx.z == 0 && op.dbias != nullptr) {
      const int i = e - 32;
      const int co = co_base + 2 * (m + TGM * (i >> 1)) + (i & 1);
      if (co < Cout) atomicAdd(&op.dbias[co], s);
    }
  }
}

template <int CO_B, int R_B, bool K1, int BW_PC>
static int launch_bww_pc(const SeistOp& op, cudaStream_t s, int sm_count) {
  constexpr int BW_PITCH = BW_PC + 4;
  const int k = op.k, S = op.stride;
  int nci_max = (R_B + k - 1) / k + 1;
  if (nci_max > op.Cin / op.groups) nci_max = op.Cin / op.groups;
  const int width = BW_PC * S + k - S;
  const int pitch = K1 ? BW_PITCH : (width | 1);
  int stage_f = (CO_B / 2) * (2 * BW_PC + 8) + nci_max * pitch;
  if (stage_f < BW_NT * 36) stage_f = BW_NT * 36;
  size_t smem = sizeof(float) * (size_t)((stage_f + 3) & ~3) + sizeof(PwOut) * CO_B + sizeof(PwChan) * (nci_max + 1) + 64 +
                (op.up_src_L > 0 ? sizeof(float) * (size_t)nci_max * (width + 4) : 0);
  // raw planes of the asynchronous gacc staging (x, dxd next to du) - unless they would cost the second resident CTA
  smem = (smem + 15) & ~(size_t)15;
  const int gx_off = (int)(smem / sizeof(float));
  const bool has_bn = op.out.bn >= 0 && op.out.g != nullptr;
  const bool need_x = has_bn || op.out_act == SEIST_OUT_SIGMOID;
  const int planes = (need_x ? 1 : 0) + ((has_bn && op.out_dxd != nullptr) ? 1 : 0);
  const size_t extra = sizeof(float) * (size_t)planes * (CO_B / 2) * (2 * BW_PC + 8);
  const bool g_async = (op.L_out & 3) == 0 && !(smem <= 113 * 1024 && smem + extra > 113 * 1024);
  if (g_async) smem += extra;
  const int R = (op.Cin / op.groups) * k;
  const int gy = op.groups * ((op.Cout / op.groups + CO_B - 1) / CO_B), gz = (R + R_B - 1) / R_B;
  const long tiles = (long)op.N * ((op.L_out + BW_PC - 1) / BW_PC);
  long gx = ((long)BWW_WAVES * sm_count + gy * gz - 1) / (gy * gz);
  if (gx > tiles) gx = tiles;
  if (gx < 1) gx = 1;
  int rc = pw_set_smem(bww_kernel<CO_B, R_B, K1, BW_PC>, smem);
  if (rc) return rc;
  bww_kernel<CO_B, R_B, K1, BW_PC><<<dim3((unsigned)gx, gy, gz), BW_NT, smem, s>>>(op, nci_max, g_async ? 1 : 0, gx_off);
  note_launch();
  return check_launch("bww");
}

template <int CO_B, int R_B, bool K1>
static int launch_bww(const SeistOp& op, cudaStream_t s, int sm_count) {
  int nci = (R_B + op.k - 1) / op.k + 1;
  if (nci > op.Cin / op.groups) nci = op.Cin / op.groups;
  // longer chunks amortise the per-chunk barriers / exposed load latency wherever the rows are long enough
  // and the staged tile still fits comfortably: 512 samples for narrow tiles, 256 for medium ones
  const int rows = CO_B + nci;
  if (rows <= 32 && op.L_out >= 2048) return launch_bww_pc<CO_B, R_B, K1, 512>(op, s, sm_count);
  if (rows <= 96 && op.L_out >= 512) return launch_bww_pc<CO_B, R_B, K1, 256>(op, s, sm_count);
  return launch_bww_pc<CO_B, R_B, K1, 128>(op, s, sm_count);
}

template <bool K1>
static int launch_bww_sel(const SeistOp& op, cudaStream_t s, int sm_count) {
  const int co = op.Cout / op.groups, R = (op.Cin / op.groups) * op.k;
  if (co <= 8) {
    if (R <= 8) return launch_bww<8, 8, K1>(op, s, sm_count);
    if (R <= 16) return launch_bww<8, 16, K1>(op, s, sm_count);
    if (R <= 32) return launch_bww<8, 32, K1>(op, s, sm_count);
    return launch_bww<8, 64, K1>(op, s, sm_count);
  }
  if (co <= 16) {
    if (R <= 8) return launch_bww<16, 8, K1>(op, s, sm_count);
    if (R <= 16) return launch_bww<16, 16, K1>(op, s, sm_count);
    if (R <= 32) return launch_bww<16, 32, K1>(op, s, sm_count);
    return launch_bww<16, 64, K1>(op, s, sm_count);
  }
  if (R <= 8) return launch_bww<32, 8, K1>(op, s, sm_count);
  if (R <= 16) return launch_bww<32, 16, K1>(op, s, sm_count);
  if (R <= 32) return launch_bww<32, 32, K1>(op, s, sm_count);
  return launch_bww<32, 64, K1>(op, s, sm_count);
}

// eligibility: dense (groups == 1), single input view unless k == 1, no pooling
bool bww_eligible(const SeistOp& op) {
  if (op.groups > 1 && ((op.Cin / op.groups) < 8 || (op.Cout / op.groups) < 8)) return false;
  if ((op.k > 1 || op.pool > 1) && op.n_in != 1) return false;
  return true;
}

int launch_bww_any(const SeistOp& op, cudaStream_t s, int sm_count) {
  if (op.k == 1 && op.stride == 1) return launch_bww_sel<true>(op, s, sm_count);
  return launch_bww_sel<false>(op, s, sm_count);
}

}  // namespace seist
