// Shared device helpers for the seist_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/seist_b200.h"

#define SEIST_ACT_NONE 0
#define SEIST_ACT_GELU 1
#define SEIST_OUT_SIGMOID 1
#define SEIST_OUT_SOFTMAX 2

namespace seist {

// ---- launch bookkeeping (api.cu) -------------------------------------------------------------
void note_launch();
int bww_waves();   // resident CTAs per SM the persistent weight-gradient kernels are sized for (SEIST_BWW_WAVES, default 2)
int env_knob(const char* name, int def);   // integer tuning knob from the environment (measurement only)
int check_launch(const char* what);
void set_error(const char* msg);

// ---- math -------------------------------------------------------------------------------------
// Two-lane fp32 helpers.  Hopper has no packed fp32 instructions, so each lane is one scalar IEEE operation; the
// _rn intrinsics keep the compiler from contracting a multiply and an add into an FMA, so the kernels compute exactly
// the sequence of roundings written here.
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 dup2(float v) { return make_float2(v, v); }

// exact-erf GELU (nn.GELU(), models/seist.py:640) with erf by Abramowitz & Stegun 7.1.26: |abs error| <= 1.5e-7, i.e. at the
// level of fp32 rounding of erff itself, in 1 rcp + 1 ex2 + 7 fma instead of erff's ~40 instructions (two polynomial
// branches).  GELU / GELU' sit in the load prologue of every kernel that consumes an activated view, where they are a large
// share of the executed instructions of the narrow layers.
__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_rcp(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_erf(float z) {
  const float a = fabsf(z);
  const float t = fast_rcp(fmaf(0.3275911f, a, 1.0f));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float e = fast_ex2(-1.4426950408889634f * a * a);
  return copysignf(fmaf(-p * t, e, 1.0f), z);
}
__device__ __forceinline__ float gelu_f(float x) { return 0.5f * x * (1.0f + fast_erf(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float gelu_grad_f(float x) {
  const float cdf = 0.5f * (1.0f + fast_erf(x * 0.70710678118654752440f));
  const float pdf = 0.39894228040143267794f * fast_ex2(-0.72134752044448170368f * x * x);
  return fmaf(x, pdf, cdf);
}
// ---- two-element versions of the element-wise math ------------------------------------------------------------------
// gelu2 is bit-identical to gelu_f per lane (same operations in the same order, the polynomial negated coefficient by
// coefficient); gelu_grad2 shares erf's exponential with the density term (exp(-z^2), z = x / sqrt 2, is exp(-x^2 / 2)),
// one MUFU less than gelu_grad_f and equal to it within 2 ulp.
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
// erf(z) per lane; e = exp(-z^2) is returned as well
__device__ __forceinline__ float2 erf2(float2 z, float2& e) {
  const float2 a = make_float2(fabsf(z.x), fabsf(z.y));
  const float2 d = fma2(dup2(0.3275911f), a, dup2(1.0f));
  const float2 t = make_float2(fast_rcp(d.x), fast_rcp(d.y));
  float2 np = fma2(dup2(-1.061405429f), t, dup2(1.453152027f));   // -p
  np = fma2(np, t, dup2(-1.421413741f));
  np = fma2(np, t, dup2(0.284496736f));
  np = fma2(np, t, dup2(-0.254829592f));
  const float2 q = mul2(mul2(dup2(-1.4426950408889634f), a), a);
  e = make_float2(fast_ex2(q.x), fast_ex2(q.y));
  const float2 r = fma2(mul2(np, t), e, dup2(1.0f));
  return make_float2(copysignf(r.x, z.x), copysignf(r.y, z.y));
}
__device__ __forceinline__ float2 gelu2(float2 x) {
  float2 e;
  const float2 erf = erf2(mul2(x, dup2(0.70710678118654752440f)), e);
  return mul2(mul2(dup2(0.5f), x), add2(dup2(1.0f), erf));
}
__device__ __forceinline__ float2 gelu_grad2(float2 x) {
  float2 e;
  const float2 erf = erf2(mul2(x, dup2(0.70710678118654752440f)), e);
  const float2 cdf = fma2(dup2(0.5f), erf, dup2(0.5f));
  return fma2(x, mul2(dup2(0.39894228040143267794f), e), cdf);
}
__device__ __forceinline__ float4 gelu4(float4 v) {
  const float2 a = gelu2(make_float2(v.x, v.y)), b = gelu2(make_float2(v.z, v.w));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ float4 gelu_grad4(float4 v) {
  const float2 a = gelu_grad2(make_float2(v.x, v.y)), b = gelu_grad2(make_float2(v.z, v.w));
  return make_float4(a.x, a.y, b.x, b.y);
}
// sc * v + sh per element
__device__ __forceinline__ float4 affine4(float4 v, float sc, float sh) {
  const float2 a = fma2(dup2(sc), make_float2(v.x, v.y), dup2(sh)), b = fma2(dup2(sc), make_float2(v.z, v.w), dup2(sh));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ float4 mul4(float4 a, float4 b) {
  const float2 lo = mul2(make_float2(a.x, a.y), make_float2(b.x, b.y)), hi = mul2(make_float2(a.z, a.w), make_float2(b.z, b.w));
  return make_float4(lo.x, lo.y, hi.x, hi.y);
}
__device__ __forceinline__ float4 scale4(float4 a, float s) { return mul4(a, make_float4(s, s, s, s)); }
__device__ __forceinline__ float4 add4(float4 a, float4 b) {
  const float2 lo = add2(make_float2(a.x, a.y), make_float2(b.x, b.y)), hi = add2(make_float2(a.z, a.w), make_float2(b.z, b.w));
  return make_float4(lo.x, lo.y, hi.x, hi.y);
}
// a * b + c per element
__device__ __forceinline__ float4 fma4(float4 a, float4 b, float4 c) {
  const float2 lo = fma2(make_float2(a.x, a.y), make_float2(b.x, b.y), make_float2(c.x, c.y));
  const float2 hi = fma2(make_float2(a.z, a.w), make_float2(b.z, b.w), make_float2(c.z, c.w));
  return make_float4(lo.x, lo.y, hi.x, hi.y);
}
__device__ __forceinline__ float4 splat4(float s) { return make_float4(s, s, s, s); }
// sum of the four elements / dot product of two quads (pairwise: (x + z) + (y + w))
__device__ __forceinline__ float sum4(float4 a) {
  const float2 s = add2(make_float2(a.x, a.y), make_float2(a.z, a.w));
  return s.x + s.y;
}
__device__ __forceinline__ float dot4(float4 a, float4 b) {
  const float2 s = fma2(make_float2(a.z, a.w), make_float2(b.z, b.w), mul2(make_float2(a.x, a.y), make_float2(b.x, b.y)));
  return s.x + s.y;
}
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + __expf(-x)); }

// ---- asynchronous global -> shared copies (LDGSTS) ---------------------------------------------------------------------
// Staging loops of the form "load, transform, store to shared" expose one memory latency per iteration unless the compiler
// can batch the loads (it cannot across the conditional GELU).  The kernels therefore copy the RAW operands with cp.async
// (every copy of a tile in flight at once, no registers held) and the issuing thread transforms its own elements in place
// after cp.async.wait_group (which orders a thread's own copies: no barrier between copy and transform).
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async16(uint32_t dst, const float* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src));
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- counter-based RNG (mirrored by oracle/plan_interp.py::rng_u64 / keep_mask) -----------------
// One splitmix64 finaliser per QUAD of consecutive element indices; element idx uses the 16-bit lane
// (idx & 3) of the hash of (idx >> 2).  A keep decision compares the lane with round(p * 65536): the drop
// probability is quantised to 2^-16 (p = 0.2 -> 0.2000122), the survivors are scaled by the exact 1/(1-p)
// like torch dropout.  Vector code paths draw four decisions from one hash (keep4).
__device__ __forceinline__ uint64_t rng_u64(uint64_t step_seed, uint32_t stream, uint64_t qidx) {
  uint64_t z = step_seed * 0xD1342543DE82EF95ull + (((uint64_t)stream << 32) | 0x9E3779B9ull);
  z += qidx * 0x9E3779B97F4A7C15ull;
  z ^= z >> 30;
  z *= 0xBF58476D1CE4E5B9ull;
  z ^= z >> 27;
  z *= 0x94D049BB133111EBull;
  z ^= z >> 31;
  return z;
}
__device__ __forceinline__ uint32_t drop_threshold(float p) {
  return (uint32_t)fminf(rintf(p * 65536.0f), 65535.0f);
}
// multiplier of the survivors, 0 for dropped elements
__device__ __forceinline__ float keep_scale(float p, uint64_t seed, uint32_t stream, uint64_t idx) {
  const uint32_t lane = (uint32_t)(rng_u64(seed, stream, idx >> 2) >> (16 * (int)(idx & 3))) & 0xFFFFu;
  return lane >= drop_threshold(p) ? 1.0f / (1.0f - p) : 0.0f;
}
// four consecutive elements idx .. idx+3, idx a multiple of 4: one hash
__device__ __forceinline__ float4 keep4(float p, uint64_t seed, uint32_t stream, uint64_t idx) {
  const uint64_t h = rng_u64(seed, stream, idx >> 2);
  const uint32_t lo = (uint32_t)h, hi = (uint32_t)(h >> 32), thr = drop_threshold(p);
  const float s = 1.0f / (1.0f - p);
  return make_float4((lo & 0xFFFFu) >= thr ? s : 0.f, (lo >> 16) >= thr ? s : 0.f, (hi & 0xFFFFu) >= thr ? s : 0.f,
                     (hi >> 16) >= thr ? s : 0.f);
}
__device__ __forceinline__ uint64_t load_seed(const uint64_t* p) { return p ? *p : 0ull; }

// ---- BatchNorm coefficient algebra (mirrored by oracle/plan_interp.py) ------------------------
__device__ __forceinline__ void bn_moments(const SeistBN& e, int c, double& mean, double& var) {
  if (e.use_batch) {
    mean = e.stat[c] / e.count;
    var = e.stat[e.C + c] / e.count - mean * mean;
    var = var > 0.0 ? var : 0.0;
  } else {
    mean = (double)e.running_mean[c];
    var = (double)e.running_var[c];
  }
}

// BN(x) = scale * x + shift, a chained second BN folded in
__device__ __forceinline__ void bn_fwd_coef(const SeistBN* tab, int bn, int c, float& scale, float& shift) {
  const SeistBN& e = tab[bn];
  double mean, var;
  bn_moments(e, c, mean, var);
  const double g1 = e.gamma[c], b1 = e.beta[c];
  const double s1 = g1 * rsqrt(var + (double)e.eps);
  const double t1 = b1 - mean * s1;
  if (e.chain >= 0) {
    const SeistBN& e2 = tab[e.chain];
    double mean2, var2;
    if (e.use_batch) {
      mean2 = b1;
      var2 = s1 * s1 * var;
    } else {
      mean2 = (double)e2.running_mean[c];
      var2 = (double)e2.running_var[c];
    }
    const double s2 = (double)e2.gamma[c] * rsqrt(var2 + (double)e2.eps);
    scale = (float)(s2 * s1);
    shift = (float)(s2 * (t1 - mean2) + (double)e2.beta[c]);
  } else {
    scale = (float)s1;
    shift = (float)t1;
  }
}

// khat = (x - mu) * istd : normalised input of the (first) BN, basis of gstat's second sum
__device__ __forceinline__ void bn_khat_coef(const SeistBN* tab, int bn, int c, float& mu, float& istd) {
  const SeistBN& e = tab[bn];
  double mean, var;
  bn_moments(e, c, mean, var);
  mu = (float)mean;
  istd = (float)rsqrt(var + (double)e.eps);
}

// d/dx = A * du + Bx * x + Cc   (du: gradient w.r.t. the BN output)
__device__ __forceinline__ void bn_bwd_coef(const SeistBN* tab, int bn, int c, float& A, float& Bx, float& Cc) {
  const SeistBN& e = tab[bn];
  double mean, var;
  bn_moments(e, c, mean, var);
  const double eps = e.eps, cnt = e.count;
  const double istd = rsqrt(var + eps);
  const double g1 = e.gamma[c];
  const double S1 = e.gstat[c], S2 = e.gstat[e.C + c];
  double a, kc, c0;
  if (e.chain < 0) {
    a = g1 * istd;
    kc = -a * S2 / cnt;
    c0 = -a * S1 / cnt;
  } else {
    const SeistBN& e2 = tab[e.chain];
    const double g2 = e2.gamma[c];
    const double vk = var * istd * istd;
    const double istd2 = rsqrt(g1 * g1 * vk + (double)e2.eps);
    const double dg1 = g2 * istd2 * S2 * (1.0 - g1 * g1 * istd2 * istd2 * vk);
    a = g1 * istd * g2 * istd2;
    kc = -g1 * istd * (g2 * istd2 * g1 * g1 * istd2 * istd2 * S2 / cnt + dg1 / cnt);
    c0 = -a * S1 / cnt;
  }
  A = (float)a;
  Bx = (float)(kc * istd);
  Cc = (float)(c0 - kc * istd * mean);
}

// ---- views ------------------------------------------------------------------------------------
// Resolve concatenated-input channel `ci` to (view index, channel inside the view).
__device__ __forceinline__ int resolve_view(const SeistOp& op, int ci, int& cv) {
  int v = 0;
  cv = ci;
#pragma unroll
  for (int i = 0; i < SEIST_MAX_IN - 1; ++i) {
    if (v == i && i + 1 < op.n_in && cv >= op.in[i].C) {
      cv -= op.in[i].C;
      v = i + 1;
    }
  }
  return v;
}

__device__ __forceinline__ const float* view_row(const SeistView& v, int n, int c) {
  return v.x + ((size_t)n * v.Ct + v.c0 + c) * (size_t)v.L;
}
__device__ __forceinline__ float* view_grad_row(const SeistView& v, int n, int c) {
  return v.g + ((size_t)n * v.Ct + v.c0 + c) * (size_t)v.L;
}
// coefficient table row of channel c of the BN applied by view v (written by the BN_PREPARE ops)
__device__ __forceinline__ const float* bn_coef_row(const SeistOp& op, int bn, int c) {
  return op.bn_table[bn].coef + 8 * (size_t)c;
}
__device__ __forceinline__ void view_coef(const SeistOp& op, const SeistView& v, int c, float& sc, float& sh) {
  if (v.bn >= 0) {
    if (op.bn_table[v.bn].inline_coef) {
      bn_fwd_coef(op.bn_table, v.bn, v.bn_c0 + c, sc, sh);     // once per channel per CTA: cheaper than a launch per BN
      return;
    }
    const float2 k = *reinterpret_cast<const float2*>(bn_coef_row(op, v.bn, v.bn_c0 + c));
    sc = k.x;
    sh = k.y;
  } else {
    sc = 1.0f;
    sh = 0.0f;
  }
}

// per-channel gradient prologue of the op's output: dOut = A*du + Bx*x + Cc + dxd (then sigmoid')
struct OutGradCoef {
  float A, Bx, Cc;
};
__device__ __forceinline__ OutGradCoef out_grad_coef(const SeistOp& op, int co) {
  OutGradCoef k;
  if (op.out.bn >= 0 && op.out.g != nullptr) {
    if (op.bn_table[op.out.bn].inline_coef) {
      bn_bwd_coef(op.bn_table, op.out.bn, op.out.bn_c0 + co, k.A, k.Bx, k.Cc);
      return k;
    }
    const float4 t = *reinterpret_cast<const float4*>(bn_coef_row(op, op.out.bn, op.out.bn_c0 + co) + 4);
    k.A = t.x;
    k.Bx = t.y;
    k.Cc = t.z;
  } else {
    k.A = 0.f;
    k.Bx = 0.f;
    k.Cc = 0.f;
  }
  return k;
}
__device__ __forceinline__ float out_grad_at(const SeistOp& op, const OutGradCoef& k, int n, int co, int l) {
  const size_t off = ((size_t)n * op.out.Ct + op.out.c0 + co) * (size_t)op.out.L + l;
  float g = 0.f;
  if (op.out_dxd != nullptr) g = op.out_dxd[off];
  const bool has_bn = (op.out.bn >= 0 && op.out.g != nullptr);
  if (has_bn || op.out_act == SEIST_OUT_SIGMOID) {
    const float x = op.out.x[off];
    if (has_bn) g += k.A * op.out.g[off] + k.Bx * x + k.Cc;
    if (op.out_act == SEIST_OUT_SIGMOID) g *= x * (1.0f - x);
  }
  return g;
}

// khat = (x - mu) * istd of the BN applied by view v
__device__ __forceinline__ void view_khat(const SeistOp& op, const SeistView& v, int c, float& mu, float& istd) {
  if (op.bn_table[v.bn].inline_coef) {
    bn_khat_coef(op.bn_table, v.bn, v.bn_c0 + c, mu, istd);
    return;
  }
  const float2 k = *reinterpret_cast<const float2*>(bn_coef_row(op, v.bn, v.bn_c0 + c) + 2);
  mu = k.x;
  istd = k.y;
}

// deposit a per-channel pair of gstat partial sums (called by one lane per warp)
__device__ __forceinline__ void gstat_add(const SeistOp& op, const SeistView& v, int c, float s1, float s2) {
  const SeistBN& e = op.bn_table[v.bn];
  atomicAdd(&e.gstat_acc[v.bn_c0 + c], (double)s1);
  atomicAdd(&e.gstat_acc[e.C + v.bn_c0 + c], (double)s2);
}

// drop factors of the epilogue: fac = delta(n) * D(n,co,l), alpha(n)
__device__ __forceinline__ float path_factor(const SeistOp& op, uint64_t seed, int n) {
  return op.p_path > 0.f ? keep_scale(op.p_path, seed, op.seed_path, (uint64_t)n) : 1.f;
}
__device__ __forceinline__ float alpha_factor(const SeistOp& op, uint64_t seed, int n) {
  return op.p_alpha > 0.f ? keep_scale(op.p_alpha, seed, op.seed_alpha, (uint64_t)n) : 1.f;
}
__device__ __forceinline__ float elem_factor(const SeistOp& op, uint64_t seed, int n, int co, int l) {
  if (op.p_elem <= 0.f) return 1.f;
  const uint64_t idx = ((uint64_t)n * op.Cout + co) * (uint64_t)op.L_out + l;
  return keep_scale(op.p_elem, seed, op.seed_elem, idx);
}


}  // namespace seist
