// Attention core of AttentionBlock (reference models/seist.py:381-388):
//   out[n, h*E+e, l] = sum_j softmax_j( (q[n,h,:,l]/sqrt(E)) . k[n,h,:,j] ) * v[n,h,e,j]
// q is (N, C, Lq), k/v are (N, C, Lk) with Lk = Lq / attn_aggr_ratio = L / 64 at every stage: 128 for L = 8192,
// 157 for 10000, 256 for 16384 (the longest window preprocess and pick_phase accept).  K and V of one (waveform,
// head) are staged through shared memory KV_CHUNK keys at a time — at most 2 x 32 x 128 floats, one chunk up to
// L = 8192, two past it — and each thread owns one query column in registers (flash-style online softmax carried
// across the chunks, no (Lq x Lk) matrix in HBM).  tests/test_gpu_attention.py checks all three kernels across
// chunk boundaries against float64.
// Lanes run along the sample axis: every global access is a coalesced channel-row segment.
#include "common.cuh"

namespace seist {

constexpr int ATT_NT = 128;
constexpr int KV_CHUNK = 128;

// Shared rows are stored per key / query: [j][K(E) | V(E)] (pitch 2E+4 floats keeps 16-byte alignment and
// spreads the transposing stores over 8 bank groups), so the thread that owns a query column reads the whole
// key as E/4 broadcast 16-byte loads and contracts it over (even, odd) feature pairs (fma2).
template <int E>
struct AttRow {
  static constexpr int PITCH = 2 * E + 4;
};

__device__ __forceinline__ float attn_keep(const SeistOp& op, uint64_t seed, int n, int h, int l, int j) {
  if (op.p_attn <= 0.f) return 1.f;
  const uint64_t idx = (((uint64_t)n * op.heads + h) * (uint64_t)op.L_out + l) * (uint64_t)op.L_in + j;
  return keep_scale(op.p_attn, seed, op.seed_attn, idx);
}
// keys j..j+3 (j a multiple of 4, Lk a multiple of 4): one hash
__device__ __forceinline__ float4 attn_keep4(const SeistOp& op, uint64_t seed, int n, int h, int l, int j) {
  const uint64_t idx = (((uint64_t)n * op.heads + h) * (uint64_t)op.L_out + l) * (uint64_t)op.L_in + j;
  return keep4(op.p_attn, seed, op.seed_attn, idx);
}

template <int E>
__device__ __forceinline__ void att_load_pairs(const float* row, float2 (&dst)[E / 2]) {
#pragma unroll
  for (int v = 0; v < E / 4; ++v) {
    const float4 t = *reinterpret_cast<const float4*>(row + 4 * v);
    dst[2 * v] = make_float2(t.x, t.y);
    dst[2 * v + 1] = make_float2(t.z, t.w);
  }
}

// stage K and V of keys j0 .. j0+KV_CHUNK of one (waveform, head) as [j][K|V]
template <int E>
__device__ __forceinline__ void att_stage_kv(const SeistOp& op, float* kv_s, int n, int h, int j0, int jn) {
  constexpr int P = AttRow<E>::PITCH;
  const SeistView &kv = op.in[1], &vv = op.in[2];
  for (int idx = threadIdx.x; idx < E * KV_CHUNK; idx += ATT_NT) {
    const int e = idx / KV_CHUNK, j = idx % KV_CHUNK;
    kv_s[j * P + e] = j < jn ? view_row(kv, n, h * E + e)[j0 + j] : 0.f;
    kv_s[j * P + E + e] = j < jn ? view_row(vv, n, h * E + e)[j0 + j] : 0.f;
  }
}

// ---- forward: grid (ceil(Lq/128), N*heads) --------------------------------------------------------
template <int E>
__global__ void __launch_bounds__(ATT_NT) att_fwd_kernel(const __grid_constant__ SeistOp op) {
  constexpr int P = AttRow<E>::PITCH;
  __shared__ __align__(16) float kv_s[KV_CHUNK * P];
  const int n = blockIdx.y / op.heads, h = blockIdx.y % op.heads;
  const int l = blockIdx.x * ATT_NT + threadIdx.x;
  const int Lq = op.L_out, Lk = op.L_in;
  const bool ok = l < Lq;
  const uint64_t seed = load_seed(op.step_seed);
  const float scale = rsqrtf((float)E);
  const SeistView& qv = op.in[0];
  const bool drop = op.p_attn > 0.f, quad = (Lk & 3) == 0;

  float2 q[E / 2], o[E / 2];
#pragma unroll
  for (int e = 0; e < E / 2; ++e) {
    q[e].x = ok ? view_row(qv, n, h * E + 2 * e)[l] * scale : 0.f;
    q[e].y = ok ? view_row(qv, n, h * E + 2 * e + 1)[l] * scale : 0.f;
    o[e] = make_float2(0.f, 0.f);
  }
  float m = -INFINITY, den = 0.f;
  for (int j0 = 0; j0 < Lk; j0 += KV_CHUNK) {
    const int jn = min(KV_CHUNK, Lk - j0);
    __syncthreads();
    att_stage_kv<E>(op, kv_s, n, h, j0, jn);
    __syncthreads();
    for (int jq = 0; jq < jn; jq += 4) {
      float kp[4] = {1.f, 1.f, 1.f, 1.f};
      if (drop && ok) {
        if (quad) {
          const float4 t = attn_keep4(op, seed, n, h, l, j0 + jq);
          kp[0] = t.x;
          kp[1] = t.y;
          kp[2] = t.z;
          kp[3] = t.w;
        } else {
#pragma unroll
          for (int u = 0; u < 4; ++u) kp[u] = (jq + u < jn) ? attn_keep(op, seed, n, h, l, j0 + jq + u) : 1.f;
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int j = jq + u;
        if (j >= jn) break;
        float2 k2[E / 2], v2[E / 2];
        att_load_pairs<E>(kv_s + j * P, k2);
        att_load_pairs<E>(kv_s + j * P + E, v2);
        float2 s2 = make_float2(0.f, 0.f);
#pragma unroll
        for (int e = 0; e < E / 2; ++e) s2 = fma2(q[e], k2[e], s2);
        const float s = s2.x + s2.y;
        if (s > m) {   // rescale only when the running maximum moves
          const float r = __expf(m - s);
          den *= r;
#pragma unroll
          for (int e = 0; e < E / 2; ++e) o[e] = mul2(o[e], dup2(r));
          m = s;
        }
        const float p = __expf(s - m);
        den += p;
        const float2 pd = dup2(p * kp[u]);
#pragma unroll
        for (int e = 0; e < E / 2; ++e) o[e] = fma2(pd, v2[e], o[e]);
      }
    }
  }
  if (ok) {
    const float inv = 1.f / den;
#pragma unroll
    for (int e = 0; e < E / 2; ++e) {
      op.out.x[((size_t)n * op.out.Ct + op.out.c0 + h * E + 2 * e) * (size_t)Lq + l] = o[e].x * inv;
      op.out.x[((size_t)n * op.out.Ct + op.out.c0 + h * E + 2 * e + 1) * (size_t)Lq + l] = o[e].y * inv;
    }
    if (op.lse) op.lse[((size_t)n * op.heads + h) * Lq + l] = m + __logf(den);
  }
}

// ---- backward w.r.t. q: grid (ceil(Lq/128), N*heads); also writes delta[l] = sum_e dO*O -------------
template <int E>
__global__ void __launch_bounds__(ATT_NT) att_bwd_q_kernel(const __grid_constant__ SeistOp op) {
  constexpr int P = AttRow<E>::PITCH;
  __shared__ __align__(16) float kv_s[KV_CHUNK * P];
  const int n = blockIdx.y / op.heads, h = blockIdx.y % op.heads;
  const int l = blockIdx.x * ATT_NT + threadIdx.x;
  const int Lq = op.L_out, Lk = op.L_in;
  const bool ok = l < Lq;
  const uint64_t seed = load_seed(op.step_seed);
  const float scale = rsqrtf((float)E);
  const SeistView& qv = op.in[0];
  const bool drop = op.p_attn > 0.f, quad = (Lk & 3) == 0;

  float2 q[E / 2], dO[E / 2], dq[E / 2];
  float delta = 0.f;
#pragma unroll
  for (int e = 0; e < E; ++e) {
    const size_t off = ((size_t)n * op.out.Ct + op.out.c0 + h * E + e) * (size_t)Lq + l;
    const float qe = ok ? view_row(qv, n, h * E + e)[l] * scale : 0.f;
    const float de = ok ? op.out_dxd[off] : 0.f;
    delta = fmaf(de, ok ? op.out.x[off] : 0.f, delta);
    if (e & 1) {
      q[e >> 1].y = qe;
      dO[e >> 1].y = de;
    } else {
      q[e >> 1].x = qe;
      dO[e >> 1].x = de;
    }
  }
#pragma unroll
  for (int e = 0; e < E / 2; ++e) dq[e] = make_float2(0.f, 0.f);
  const float lse = ok ? op.lse[((size_t)n * op.heads + h) * Lq + l] : 0.f;
  if (ok) op.delta[((size_t)n * op.heads + h) * Lq + l] = delta;
  for (int j0 = 0; j0 < Lk; j0 += KV_CHUNK) {
    const int jn = min(KV_CHUNK, Lk - j0);
    __syncthreads();
    att_stage_kv<E>(op, kv_s, n, h, j0, jn);
    __syncthreads();
    for (int jq = 0; jq < jn; jq += 4) {
      float kp[4] = {1.f, 1.f, 1.f, 1.f};
      if (drop && ok) {
        if (quad) {
          const float4 t = attn_keep4(op, seed, n, h, l, j0 + jq);
          kp[0] = t.x;
          kp[1] = t.y;
          kp[2] = t.z;
          kp[3] = t.w;
        } else {
#pragma unroll
          for (int u = 0; u < 4; ++u) kp[u] = (jq + u < jn) ? attn_keep(op, seed, n, h, l, j0 + jq + u) : 1.f;
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int j = jq + u;
        if (j >= jn) break;
        float2 k2[E / 2], v2[E / 2];
        att_load_pairs<E>(kv_s + j * P, k2);
        att_load_pairs<E>(kv_s + j * P + E, v2);
        float2 s2 = make_float2(0.f, 0.f), dp2 = make_float2(0.f, 0.f);
#pragma unroll
        for (int e = 0; e < E / 2; ++e) {
          s2 = fma2(q[e], k2[e], s2);
          dp2 = fma2(dO[e], v2[e], dp2);
        }
        const float p = __expf((s2.x + s2.y) - lse);
        const float2 ds = dup2(p * ((dp2.x + dp2.y) * kp[u] - delta));
#pragma unroll
        for (int e = 0; e < E / 2; ++e) dq[e] = fma2(ds, k2[e], dq[e]);
      }
    }
  }
  if (ok && qv.g != nullptr) {
#pragma unroll
    for (int e = 0; e < E; ++e) {
      float* g = view_grad_row(qv, n, h * E + e) + l;
      const float val = ((e & 1) ? dq[e >> 1].y : dq[e >> 1].x) * scale;
      if (qv.accum) *g += val; else *g = val;
    }
  }
}

// ---- backward w.r.t. k, v: grid (ceil(Lk/128), N*heads); one thread per key, loop over queries ------
template <int E>
__global__ void __launch_bounds__(ATT_NT) att_bwd_kv_kernel(const __grid_constant__ SeistOp op) {
  constexpr int QC = 64;
  constexpr int P = AttRow<E>::PITCH;
  __shared__ __align__(16) float qd_s[QC * P];   // [i][q*scale (E) | dO (E)]
  __shared__ float lse_s[QC];
  __shared__ float dl_s[QC];
  const int n = blockIdx.y / op.heads, h = blockIdx.y % op.heads;
  const int j = blockIdx.x * ATT_NT + threadIdx.x;
  const int Lq = op.L_out, Lk = op.L_in;
  const bool ok = j < Lk;
  const uint64_t seed = load_seed(op.step_seed);
  const float scale = rsqrtf((float)E);
  const SeistView &qv = op.in[0], &kv = op.in[1], &vv = op.in[2];

  float2 kk[E / 2], vj[E / 2], dk[E / 2], dv[E / 2];
#pragma unroll
  for (int e = 0; e < E / 2; ++e) {
    kk[e].x = ok ? view_row(kv, n, h * E + 2 * e)[j] : 0.f;
    kk[e].y = ok ? view_row(kv, n, h * E + 2 * e + 1)[j] : 0.f;
    vj[e].x = ok ? view_row(vv, n, h * E + 2 * e)[j] : 0.f;
    vj[e].y = ok ? view_row(vv, n, h * E + 2 * e + 1)[j] : 0.f;
    dk[e] = make_float2(0.f, 0.f);
    dv[e] = make_float2(0.f, 0.f);
  }
  for (int l0 = 0; l0 < Lq; l0 += QC) {
    const int ln = min(QC, Lq - l0);
    __syncthreads();
    for (int idx = threadIdx.x; idx < E * QC; idx += ATT_NT) {
      const int e = idx / QC, i = idx % QC;
      const size_t off = ((size_t)n * op.out.Ct + op.out.c0 + h * E + e) * (size_t)Lq + l0 + i;
      qd_s[i * P + e] = i < ln ? view_row(qv, n, h * E + e)[l0 + i] * scale : 0.f;
      qd_s[i * P + E + e] = i < ln ? op.out_dxd[off] : 0.f;
    }
    for (int i = threadIdx.x; i < QC; i += ATT_NT) {
      lse_s[i] = i < ln ? op.lse[((size_t)n * op.heads + h) * Lq + l0 + i] : 0.f;
      dl_s[i] = i < ln ? op.delta[((size_t)n * op.heads + h) * Lq + l0 + i] : 0.f;
    }
    __syncthreads();
    for (int i = 0; i < ln; ++i) {
      float2 q2[E / 2], d2[E / 2];
      att_load_pairs<E>(qd_s + i * P, q2);
      att_load_pairs<E>(qd_s + i * P + E, d2);
      float2 s2 = make_float2(0.f, 0.f), dp2 = make_float2(0.f, 0.f);
#pragma unroll
      for (int e = 0; e < E / 2; ++e) {
        s2 = fma2(q2[e], kk[e], s2);
        dp2 = fma2(d2[e], vj[e], dp2);
      }
      const float p = __expf((s2.x + s2.y) - lse_s[i]);
      const float keep = ok ? attn_keep(op, seed, n, h, l0 + i, j) : 1.f;
      const float2 pd = dup2(p * keep);
      const float2 ds = dup2(p * ((dp2.x + dp2.y) * keep - dl_s[i]));
#pragma unroll
      for (int e = 0; e < E / 2; ++e) {
        dv[e] = fma2(pd, d2[e], dv[e]);
        dk[e] = fma2(ds, q2[e], dk[e]);   // q already carries 1/sqrt(E)
      }
    }
  }
  if (ok) {
#pragma unroll
    for (int e = 0; e < E; ++e) {
      if (kv.g != nullptr) {
        float* g = view_grad_row(kv, n, h * E + e) + j;
        const float val = (e & 1) ? dk[e >> 1].y : dk[e >> 1].x;
        if (kv.accum) *g += val; else *g = val;
      }
      if (vv.g != nullptr) {
        float* g = view_grad_row(vv, n, h * E + e) + j;
        const float val = (e & 1) ? dv[e >> 1].y : dv[e >> 1].x;
        if (vv.accum) *g += val; else *g = val;
      }
    }
  }
}

#define ATT_DISPATCH(KERNEL, GRIDX)                                         \
  {                                                                         \
    const int E = op.Cout / op.heads;                                       \
    dim3 grid((GRIDX + ATT_NT - 1) / ATT_NT, op.N * op.heads);              \
    switch (E) {                                                            \
      case 8: KERNEL<8><<<grid, ATT_NT, 0, s>>>(op); break;                 \
      case 16: KERNEL<16><<<grid, ATT_NT, 0, s>>>(op); break;               \
      case 32: KERNEL<32><<<grid, ATT_NT, 0, s>>>(op); break;               \
      default: set_error("attention: head_dim must be 8, 16 or 32"); return -3; \
    }                                                                       \
    note_launch();                                                          \
  }

int launch_att_fwd(const SeistOp& op, cudaStream_t s) {
  ATT_DISPATCH(att_fwd_kernel, op.L_out)
  return check_launch("att_fwd");
}
int launch_att_bwd_q(const SeistOp& op, cudaStream_t s) {
  ATT_DISPATCH(att_bwd_q_kernel, op.L_out)
  return check_launch("att_bwd_q");
}
int launch_att_bwd_kv(const SeistOp& op, cudaStream_t s) {
  ATT_DISPATCH(att_bwd_kv_kernel, op.L_in)
  return check_launch("att_bwd_kv");
}

}  // namespace seist
