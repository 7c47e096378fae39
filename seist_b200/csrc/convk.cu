// Dense (groups == 1) k-tap convolutions: the composed stem paths (k = 5..19, stride 1/2, reference
// models/seist.py:124-155) and the up-sampling head (k = 7/11 behind F.interpolate(linear), :536,:566).
//
// Tile: 256 threads = WC channel-warps x WP sample-warps; a thread owns 4 CONSECUTIVE output samples x 8
// output channels.  The (channel, sample) input tile with halo is staged once per 8-channel chunk with
// BN-apply / GELU / linear up-sampling / zero padding evaluated on the way in; per reduction channel a
// thread pulls its sliding window (3*S + K samples) with 16-byte shared loads and reuses every window
// element for up to K taps x 8 channels (K and S are template parameters so the window lives in
// registers).  The same engine run with flipped/transposed weights over the BN-backward-combined output
// gradient is the data gradient (stride 1).  The weight gradient keeps lanes on the sample axis: a warp
// owns a (4 co) x (TCI ci) x K tile of dW in registers and reduces it over lanes once per CTA lifetime.
#include <algorithm>
#include "common.cuh"
#include "conv_common.cuh"

namespace seist {

constexpr int CK_NT = 256;
constexpr int CK_CIC = 8;

__device__ __forceinline__ float4 lds4(const float* p) { return *reinterpret_cast<const float4*>(p); }

template <int K, int S>
struct CkWin {
  static constexpr int WIN = 3 * S + K;
  static constexpr int NV = (WIN + 3) / 4;
};

// acc[c][j] += sum_t w[t][c] * win[j*S + t] for one reduction channel
// channel pairs ride the two lanes of fma2; ck_acc reads channel c, sample j of a [4][4] pair tile
__device__ __forceinline__ float ck_acc(const float2 (&acc)[4][4], int c, int j) { return (c & 1) ? acc[c >> 1][j].y : acc[c >> 1][j].x; }

template <int K, int S>
__device__ __forceinline__ void ck_accumulate(const float* irow, const float* wrow, int wstride, float2 (&acc)[4][4]) {
  constexpr int NV = CkWin<K, S>::NV;
  float win[NV * 4];
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const float4 q = lds4(irow + 4 * v);
    win[4 * v] = q.x;
    win[4 * v + 1] = q.y;
    win[4 * v + 2] = q.z;
    win[4 * v + 3] = q.w;
  }
#pragma unroll
  for (int t = 0; t < K; ++t) {
    const float4 w0 = lds4(wrow + t * wstride), w1 = lds4(wrow + t * wstride + 4);
    const float2 w[4] = {make_float2(w0.x, w0.y), make_float2(w0.z, w0.w), make_float2(w1.x, w1.y), make_float2(w1.z, w1.w)};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 v = dup2(win[j * S + t]);
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[c][j] = fma2(w[c], v, acc[c][j]);
    }
  }
}

// weights of one reduction chunk, [r][t][col] (zero padded), asynchronous 4-byte gathers
template <int K>
__device__ __forceinline__ void ck_issue_weights_fwd(const SeistOp& op, float* w_s, int CO_B, int co_base, int co_end, int gs_in,
                                                     int ci0, int cic) {
  const uint32_t wa = smem_addr(w_s);
  for (int idx = threadIdx.x; idx < CK_CIC * K * CO_B; idx += CK_NT) {
    const int col = idx % CO_B, rest = idx / CO_B;
    const int t = rest % K, r = rest / K;
    const int co = co_base + col;
    if (r < cic && co < co_end) cp_async4(wa + 4 * idx, op.W + ((size_t)co * gs_in + ci0 + r) * K + t);
    else w_s[idx] = 0.f;
  }
}

// ================================================================================================
// forward
// ================================================================================================
template <int K, int S, int NBUF>
__global__ void __launch_bounds__(CK_NT, 3) convk_fwd_kernel(const __grid_constant__ SeistOp op, const int WC) {
  extern __shared__ __align__(16) float ck_smem[];
  const int WP = 8 / WC, CO_B = 8 * WC, TLo = 128 * WP;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wc = warp % WC, wp = warp / WC;
  const int gs_in = op.Cin / op.groups, gs_out = op.Cout / op.groups;
  const int tpg = (gs_out + CO_B - 1) / CO_B;          // output-channel tiles per group
  const int grp = blockIdx.z / tpg;
  const int n = blockIdx.y, l0 = blockIdx.x * TLo, co_base = grp * gs_out + (blockIdx.z - grp * tpg) * CO_B;
  const int co_end = (grp + 1) * gs_out;               // channels of this group only
  const int ci_grp = grp * gs_in;
  const int width = TLo * S + K - S;
  const int pitch = ((width + 3) & ~3) + 4;
  // Shared memory: raw operands of reduction chunk c + 1 are copied asynchronously while chunk c is being accumulated
  // (NBUF == 2: plain rows are double buffered and transformed in place; up-sampled rows double buffer the SOURCE window
  // and interpolate into the single in_s); NBUF == 1 where two stages do not fit: copies of a chunk all in flight at once.
  const bool up = op.up_src_L > 0;
  const int spitch = width + 4;
  const int in_f = CK_CIC * pitch, w_f = CK_CIC * K * CO_B, src_f = up ? CK_CIC * spitch : 0;
  float* red_s = ck_smem;                              // [8 warps][16]
  float* in_s = ck_smem + 8 * 16;                      // [NBUF (1 if up)][CIC][pitch]
  float* w_s = in_s + (up ? 1 : NBUF) * in_f;          // [NBUF][CIC][K][CO_B]
  float* src_s = w_s + NBUF * w_f;                     // [NBUF][CIC][width+4] (up-sampled input only)
  const int Lsrc = op.in[0].L;
  const float ratio = up ? (float)Lsrc / (float)op.L_in : 1.f;
  const int p_base = l0 * S - op.pad_left;
  int i_lo = 0, count = 0;
  if (up) upsample_window(op, p_base, width, spitch, Lsrc, ratio, i_lo, count);

  float2 acc[4][4];
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[c][j] = make_float2(0.f, 0.f);

  const int nchunks = (gs_in + CK_CIC - 1) / CK_CIC;
  auto issue = [&](int c) {
    const int b = (NBUF == 2) ? (c & 1) : 0;
    const int ci0 = c * CK_CIC, cic = min(CK_CIC, gs_in - ci0);
    if (up) src_issue(op, n, ci_grp + ci0, cic, src_s + b * src_f, spitch, i_lo, count);
    else rows_issue_plain(op, n, ci_grp + ci0, cic, cic, in_s + b * in_f, pitch, width, p_base);
    ck_issue_weights_fwd<K>(op, w_s + b * w_f, CO_B, co_base, co_end, gs_in, ci0, cic);
    cp_async_commit();
  };
  if (NBUF == 2) issue(0);
  for (int c = 0; c < nchunks; ++c) {
    const int b = (NBUF == 2) ? (c & 1) : 0;
    const int ci0 = c * CK_CIC, cic = min(CK_CIC, gs_in - ci0);
    if (NBUF == 1) issue(c);
    cp_async_wait<0>();
    if (up) src_transform(op, n, ci_grp + ci0, cic, src_s + b * src_f, spitch, count);
    else rows_transform_plain(op, n, ci_grp + ci0, cic, in_s + b * in_f, pitch, width, p_base);
    __syncthreads();                                   // chunk c is staged; everybody is done with chunk c - 1
    if (NBUF == 2 && c + 1 < nchunks) issue(c + 1);
    const float* in_c = up ? in_s : in_s + b * in_f;
    if (up) {
      rows_interpolate(op, cic, in_s, pitch, width, p_base, src_s + b * src_f, spitch, i_lo, Lsrc, ratio);
      __syncthreads();
    }
    const float* ib = in_c + (wp * 128 + 4 * lane) * S;
    const float* wb = w_s + b * w_f + wc * 8;
    for (int r = 0; r < cic; ++r) ck_accumulate<K, S>(ib + r * pitch, wb + r * K * CO_B, CO_B, acc);
    if (NBUF == 1) __syncthreads();
  }

  // ---- epilogue ----------------------------------------------------------------------------------
  const uint64_t seed = load_seed(op.step_seed);
  const float pf = path_factor(op, seed, n), af = alpha_factor(op, seed, n);
  const bool stats = (op.out.bn >= 0) && op.bn_table[op.out.bn >= 0 ? op.out.bn : 0].use_batch;
  const int lq = l0 + wp * 128 + 4 * lane;
  const bool vec = (op.L_out & 3) == 0;
  float st[16];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int co = co_base + wc * 8 + c;
    float s1 = 0.f, s2 = 0.f;
    if (co < co_end) {
      const float b = op.bias ? op.bias[co] : 0.f;
      float asc = 1.f, ash = 0.f, bsc = 1.f, bsh = 0.f;
      const float *ra = nullptr, *rb = nullptr;
      if (op.res_a.C > 0) {
        view_coef(op, op.res_a, co, asc, ash);
        ra = view_row(op.res_a, n, co);
      }
      if (op.res_b.C > 0) {
        view_coef(op, op.res_b, co, bsc, bsh);
        rb = view_row(op.res_b, n, co);
      }
      float* orow = op.out.x + ((size_t)n * op.out.Ct + op.out.c0 + co) * (size_t)op.L_out;
      float r[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int l = lq + j;
        float v = 0.f;
        if (l < op.L_out) {
          v = (ck_acc(acc, c, j) + b) * pf * elem_factor(op, seed, n, co, l);
          if (ra) v += fmaf(asc, ra[l], ash);
          v *= af;
          if (rb) v += fmaf(bsc, rb[l], bsh);
          if (op.out_act == SEIST_OUT_SIGMOID) v = sigmoid_f(v);
          s1 += v;
          s2 = fmaf(v, v, s2);
        }
        r[j] = v;
      }
      if (vec && lq + 3 < op.L_out) {
        *reinterpret_cast<float4*>(orow + lq) = make_float4(r[0], r[1], r[2], r[3]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (lq + j < op.L_out) orow[lq + j] = r[j];
      }
    }
    st[2 * c] = s1;
    st[2 * c + 1] = s2;
  }
  if (stats) {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float s = warp_sum(st[i]);
      if (lane == 0) red_s[warp * 16 + i] = s;
    }
    __syncthreads();
    for (int idx = tid; idx < WC * 16; idx += CK_NT) {
      const int w0 = idx / 16, i = idx % 16;
      float s = 0.f;
      for (int p = 0; p < WP; ++p) s += red_s[(p * WC + w0) * 16 + i];
      const int co = co_base + w0 * 8 + (i >> 1);
      if (co < co_end) {
        const SeistBN& e = op.bn_table[op.out.bn];
        atomicAdd(&e.stat_acc[(i & 1) * e.C + op.out.bn_c0 + co], (double)s);
      }
    }
  }
}

// ================================================================================================
// backward (data):  d in[ci][p] = sum_{co,t} W[co][ci][t] gacc[co][(p + pad_left - t) / S]
//   S = 1: the forward engine over the combined output gradient with flipped/transposed weights.
//   S = 2 (pad_left even): input positions split by parity, p = 2u + r.  Parity r only meets the taps
//     t = r + 2s, so each parity is a stride-1 correlation of gacc with a sub-filter of KE = (K+1)/2 taps
//     (the odd one padded with a zero tap so that both share one window): the engine runs with 8 "virtual"
//     channels per warp = 4 input channels x 2 parities, and a thread that owns 4 consecutive u writes 8
//     consecutive input samples per channel.
// ================================================================================================
template <int K, int S, int NBUF>
__global__ void __launch_bounds__(CK_NT, 3) convk_bwd_data_kernel(const __grid_constant__ SeistOp op, const int WC, const int NRAW) {
  extern __shared__ __align__(16) float ck_smem[];
  constexpr int KE = S == 2 ? (K + 1) / 2 : K;          // taps of the stride-1 engine
  constexpr int CPW = S == 2 ? 4 : 8;                   // real input channels per warp
  const int WP = 8 / WC, CI_B = CPW * WC, VC_B = 8 * WC, TLo = 128 * WP;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wc = warp % WC, wp = warp / WC;
  const int gs_in = op.Cin / op.groups, gs_out = op.Cout / op.groups;
  const int tpg = (gs_in + CI_B - 1) / CI_B;
  const int grp = blockIdx.z / tpg;
  const int n = blockIdx.y, p0 = blockIdx.x * TLo, ci_base = grp * gs_in + (blockIdx.z - grp * tpg) * CI_B;
  const int ci_end = (grp + 1) * gs_in;
  const int co_grp = grp * gs_out;
  const int width = TLo + KE - 1;
  const int pitch = ((width + 3) & ~3) + 4;
  // Shared memory: the raw operands of the output-gradient rows (du | x | dxd as the op needs them: NRAW planes) of
  // chunk c + 1 are copied asynchronously while chunk c is accumulated (NBUF == 2), and combined IN PLACE into plane 0
  // (BN backward, sigmoid', drop factors) by the thread that copied them.
  const bool has_bn = (op.out.bn >= 0 && op.out.g != nullptr);
  const bool need_x = has_bn || op.out_act == SEIST_OUT_SIGMOID;
  const int z_f = CK_CIC * pitch, w_f = CK_CIC * KE * VC_B;
  float* red_s = ck_smem;                              // [8][16]
  float* z_s = ck_smem + 8 * 16;                       // [NBUF][NRAW][CIC][pitch]
  float* w_s = z_s + NBUF * NRAW * z_f;                // [NBUF][CIC][KE][VC_B]
  const uint64_t seed = load_seed(op.step_seed);
  const float pf = path_factor(op, seed, n) * alpha_factor(op, seed, n);
  const int m_base = p0 + op.pad_left / S - (KE - 1);  // output-sample coordinate of z_s[.][0]
  const int pos_lo = max(0, -m_base), pos_hi = min(width, op.L_out - m_base);   // valid positions [pos_lo, pos_hi)
  const float* src0 = has_bn ? op.out.g : op.out_dxd;  // plane 0 (nullptr: zeros)
  const float* src2 = has_bn ? op.out_dxd : nullptr;   // plane 2

  float2 acc[4][4];
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[c][j] = make_float2(0.f, 0.f);

  const int nchunks = (gs_out + CK_CIC - 1) / CK_CIC;
  auto issue = [&](int c) {
    const int b = (NBUF == 2) ? (c & 1) : 0;
    const int co0 = c * CK_CIC, coc = min(CK_CIC, gs_out - co0);
    float* zb = z_s + b * NRAW * z_f;
    for (int r = warp; r < coc; r += CK_NT / 32) {
      const size_t row = ((size_t)n * op.out.Ct + op.out.c0 + co_grp + co0 + r) * (size_t)op.out.L + m_base;
      float* d = zb + r * pitch;
      const uint32_t da = smem_addr(d);
      for (int pos = lane; pos < width; pos += 32) {
        if (pos >= pos_lo && pos < pos_hi) {
          if (src0) cp_async4(da + 4 * pos, src0 + row + pos);
          else d[pos] = 0.f;
          if (need_x) cp_async4(da + 4 * (z_f + pos), op.out.x + row + pos);
          if (src2) cp_async4(da + 4 * (2 * z_f + pos), src2 + row + pos);
        } else {
          d[pos] = 0.f;
        }
      }
    }
    // flipped + transposed weights: w_s[(r*KE + tf)*VC_B + col] = W[co0+r][ci(col)][t(tf, parity(col))]
    float* wb = w_s + b * w_f;
    const uint32_t wa = smem_addr(wb);
    for (int idx = tid; idx < CK_CIC * KE * VC_B; idx += CK_NT) {
      const int col = idx % VC_B, rest = idx / VC_B;
      const int tf = rest % KE, r = rest / KE;
      const int ci = ci_base + (S == 2 ? (col >> 1) : col);
      const int t = S == 2 ? (col & 1) + 2 * (KE - 1 - tf) : (K - 1 - tf);
      if (r < coc && ci < ci_end && t < K)
        cp_async4(wa + 4 * idx, op.W + ((size_t)(co_grp + co0 + r) * gs_in + (ci - grp * gs_in)) * K + t);
      else
        wb[idx] = 0.f;
    }
    cp_async_commit();
  };
  auto combine = [&](int c) {
    const int b = (NBUF == 2) ? (c & 1) : 0;
    const int co0 = c * CK_CIC, coc = min(CK_CIC, gs_out - co0);
    float* zb = z_s + b * NRAW * z_f;
    const bool scale_only = !need_x;
    if (scale_only && pf == 1.f && op.p_elem <= 0.f) return;   // plane 0 already holds the gradient
    for (int r = warp; r < coc; r += CK_NT / 32) {
      const int co = co_grp + co0 + r;
      const OutGradCoef kc = out_grad_coef(op, co);
      float* d = zb + r * pitch;
      for (int pos = lane; pos < pos_hi; pos += 32) {     // (scalar)
        if (pos < pos_lo) continue;
        float g = d[pos];
        if (need_x) {
          const float x = d[z_f + pos];
          if (has_bn) {
            g = fmaf(kc.A, g, fmaf(kc.Bx, x, kc.Cc));
            if (src2) g += d[2 * z_f + pos];
          }
          if (op.out_act == SEIST_OUT_SIGMOID) g *= x * (1.0f - x);
        }
        g *= pf;
        if (op.p_elem > 0.f) g *= elem_factor(op, seed, n, co, m_base + pos);
        d[pos] = g;
      }
    }
  };
  if (NBUF == 2) issue(0);
  for (int c = 0; c < nchunks; ++c) {
    const int b = (NBUF == 2) ? (c & 1) : 0;
    const int coc = min(CK_CIC, gs_out - c * CK_CIC);
    if (NBUF == 1) issue(c);
    cp_async_wait<0>();
    combine(c);
    __syncthreads();                                   // chunk c is staged; everybody is done with chunk c - 1
    if (NBUF == 2 && c + 1 < nchunks) issue(c + 1);
    const float* zb = z_s + b * NRAW * z_f + wp * 128 + 4 * lane;
    const float* wb = w_s + b * w_f + wc * 8;
    for (int r = 0; r < coc; ++r) ck_accumulate<KE, 1>(zb + r * pitch, wb + r * KE * VC_B, VC_B, acc);
    if (NBUF == 1) __syncthreads();
  }

  // ---- route to the source view ----------------------------------------------------------------------
  const int Lsrc = op.in[0].L;
  const float ratio = op.up_src_L > 0 ? (float)Lsrc / (float)op.L_in : 1.f;
  const int pq = p0 + wp * 128 + 4 * lane;
  float st[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) st[i] = 0.f;
  // fast path (whole quads inside the row, no up-sampling): 16-byte accesses, and the loads of a batch of
  // channels (x for khat / GELU', the old gradient when accumulating) are all issued before its first store
  const int pos0 = S == 2 ? 2 * pq : pq;
  const bool fast = op.up_src_L == 0 && (op.L_in & 3) == 0 && pos0 + 4 * S - 1 < op.L_in;
  if (fast) {
    const SeistView& v = op.in[0];          // convk ops have a single input view
    if (v.g != nullptr) {
      constexpr int NV = S == 2 ? 2 : 1;    // float4 per real channel
      constexpr int CB = S == 2 ? 2 : 4;    // real channels per batch (4 x-loads + 4 old-loads in flight)
      const bool need_x = v.act == SEIST_ACT_GELU || v.bn >= 0;
#pragma unroll
      for (int kb = 0; kb < CPW; kb += CB) {
        float4 xv[CB * NV], ov[CB * NV];
#pragma unroll
        for (int u = 0; u < CB; ++u) {
          const int ci = min(ci_base + wc * CPW + kb + u, ci_end - 1);
          const size_t off = ((size_t)n * v.Ct + v.c0 + ci) * (size_t)v.L + pos0;
#pragma unroll
          for (int q = 0; q < NV; ++q) {
            xv[u * NV + q] = need_x ? __ldg(reinterpret_cast<const float4*>(v.x + off) + q) : make_float4(0.f, 0.f, 0.f, 0.f);
            ov[u * NV + q] = v.accum ? *(reinterpret_cast<const float4*>(v.g + off) + q) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
#pragma unroll
        for (int u = 0; u < CB; ++u) {
          const int k = kb + u;
          const int ci = ci_base + wc * CPW + k;
          if (ci >= ci_end) continue;
          float sc, sh, mu = 0.f, istd = 0.f;
          view_coef(op, v, ci, sc, sh);
          if (v.bn >= 0) view_khat(op, v, ci, mu, istd);
          const size_t off = ((size_t)n * v.Ct + v.c0 + ci) * (size_t)v.L + pos0;
#pragma unroll
          for (int q = 0; q < NV; ++q) {
            const float4 x4 = xv[u * NV + q], o4 = ov[u * NV + q];
            const float xs[4] = {x4.x, x4.y, x4.z, x4.w};
            const float os[4] = {o4.x, o4.y, o4.z, o4.w};
            float g[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              // S = 1: element e is sample j = e of channel k; S = 2: element 4q+e is (j, parity) = ((4q+e)>>1, e&1)
              const int c = S == 2 ? 2 * k + (e & 1) : k;
              const int j = S == 2 ? (4 * q + e) >> 1 : e;
              float gv = ck_acc(acc, c, j);
              if (v.act == SEIST_ACT_GELU) gv *= gelu_grad_f(fmaf(sc, xs[e], sh));
              st[2 * c] += gv;
              st[2 * c + 1] = fmaf(gv, (xs[e] - mu) * istd, st[2 * c + 1]);
              g[e] = gv + os[e];
            }
            *(reinterpret_cast<float4*>(v.g + off) + q) = make_float4(g[0], g[1], g[2], g[3]);
          }
        }
      }
    }
  } else if (S == 1 && op.up_src_L > 0 && 2 * Lsrc == op.L_in && (op.L_in & 3) == 0) {
    // exact x2 linear up-sampling (the dpk head, reference models/seist.py:566): the quad p = 4m .. 4m+3 only touches
    // the sources 2m-1 .. 2m+2 with the fixed weights (.25 | .75 .75 .25 | .25 .75 .75 | .25).  Every lane owns the
    // sources 2m, 2m+1: the two outer contributions travel to the neighbouring lanes by shuffle, the activation
    // derivative and the BN sums are evaluated once per SOURCE sample, and 2 (+1 at a warp edge) atomics per
    // channel replace 8 (the target is zero-initialised by the preceding ZERO op).
    const SeistView& v = op.in[0];
    if (v.g != nullptr) {
      const bool inside = pq < op.L_in;
      const int m2 = pq >> 1;                               // source index 2m
      const bool first = pq == 0, last = pq + 4 >= op.L_in;
      // the source samples of all 8 channels first: one exposed memory latency instead of one per channel
      float2 x2v[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int ci = ci_base + wc * 8 + c;
        x2v[c] = (inside && ci < ci_end) ? *reinterpret_cast<const float2*>(view_row(v, n, ci) + m2) : make_float2(0.f, 0.f);
      }
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int ci = ci_base + wc * 8 + c;
        const bool live = ci < ci_end;                      // warp-uniform
        const float d0 = inside && live ? ck_acc(acc, c, 0) : 0.f, d1 = inside && live ? ck_acc(acc, c, 1) : 0.f;
        const float d2 = inside && live ? ck_acc(acc, c, 2) : 0.f, d3 = inside && live ? ck_acc(acc, c, 3) : 0.f;
        float ga = 0.25f * d0, ge = 0.25f * d3;             // to 2m-1 / 2m+2
        float gb = 0.75f * (d0 + d1) + 0.25f * d2, gc = 0.25f * d1 + 0.75f * (d2 + d3);
        if (first) {
          gb += ga;
          ga = 0.f;
        }
        if (last) {
          gc += ge;
          ge = 0.f;
        }
        const float from_prev = __shfl_up_sync(0xffffffffu, ge, 1), from_next = __shfl_down_sync(0xffffffffu, ga, 1);
        if (lane > 0) gb += from_prev;
        if (lane < 31) gc += from_next;
        if (!live || !inside) continue;
        float sc, sh, mu = 0.f, istd = 0.f;
        view_coef(op, v, ci, sc, sh);
        if (v.bn >= 0) view_khat(op, v, ci, mu, istd);
        const float* xr = view_row(v, n, ci);
        float* gr = view_grad_row(v, n, ci);
        const float2 x2 = x2v[c];
        if (v.act == SEIST_ACT_GELU) {
          gb *= gelu_grad_f(fmaf(sc, x2.x, sh));
          gc *= gelu_grad_f(fmaf(sc, x2.y, sh));
        }
        atomicAdd(&gr[m2], gb);
        atomicAdd(&gr[m2 + 1], gc);
        float s1 = gb + gc;
        float s2 = fmaf(gb, (x2.x - mu) * istd, gc * ((x2.y - mu) * istd));
        if (lane == 0 && !first) {                           // 2m-1 belongs to the last lane of another warp
          const float xa = xr[m2 - 1];
          if (v.act == SEIST_ACT_GELU) ga *= gelu_grad_f(fmaf(sc, xa, sh));
          atomicAdd(&gr[m2 - 1], ga);
          s1 += ga;
          s2 = fmaf(ga, (xa - mu) * istd, s2);
        }
        if (lane == 31 && !last) {                           // 2m+2 belongs to the first lane of another warp
          const float xe = xr[m2 + 2];
          if (v.act == SEIST_ACT_GELU) ge *= gelu_grad_f(fmaf(sc, xe, sh));
          atomicAdd(&gr[m2 + 2], ge);
          s1 += ge;
          s2 = fmaf(ge, (xe - mu) * istd, s2);
        }
        st[2 * c] = s1;
        st[2 * c + 1] = s2;
      }
    }
  } else
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int ci = ci_base + wc * CPW + (S == 2 ? (c >> 1) : c);
    float s1 = 0.f, s2 = 0.f;
    if (ci < ci_end) {
      int cv;
      const int vi = resolve_view(op, ci, cv);
      const SeistView& v = op.in[vi];
      if (v.g != nullptr) {
        float sc, sh, mu = 0.f, istd = 0.f;
        view_coef(op, v, cv, sc, sh);
        if (v.bn >= 0) view_khat(op, v, cv, mu, istd);
        const float* xr = view_row(v, n, cv);
        float* gr = view_grad_row(v, n, cv);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int p = S == 2 ? 2 * (pq + j) + (c & 1) : pq + j;
          if (p >= op.L_in) continue;
          const float d = ck_acc(acc, c, j);
          if (op.up_src_L > 0) {
            int i0, i1;
            float lam;
            upsample_coords(p, ratio, Lsrc, i0, i1, lam);
            const float x0 = xr[i0], x1 = xr[i1];
            float g0 = d * (1.f - lam), g1 = d * lam;
            if (v.act == SEIST_ACT_GELU) {
              g0 *= gelu_grad_f(fmaf(sc, x0, sh));
              g1 *= gelu_grad_f(fmaf(sc, x1, sh));
            }
            atomicAdd(&gr[i0], g0);
            atomicAdd(&gr[i1], g1);
            s1 += g0 + g1;
            s2 = fmaf(g0, (x0 - mu) * istd, s2);
            s2 = fmaf(g1, (x1 - mu) * istd, s2);
          } else {
            const float x = xr[p];
            float g = d;
            if (v.act == SEIST_ACT_GELU) g *= gelu_grad_f(fmaf(sc, x, sh));
            if (v.accum) gr[p] += g; else gr[p] = g;
            s1 += g;
            s2 = fmaf(g, (x - mu) * istd, s2);
          }
        }
      }
    }
    st[2 * c] = s1;
    st[2 * c + 1] = s2;
  }
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const float s = warp_sum(st[i]);
    if (lane == 0) red_s[warp * 16 + i] = s;
  }
  __syncthreads();
  for (int idx = tid; idx < WC * 16; idx += CK_NT) {
    const int w0 = idx / 16, i = idx % 16;
    float s = 0.f;
    for (int p = 0; p < WP; ++p) s += red_s[(p * WC + w0) * 16 + i];
    const int ci = ci_base + w0 * CPW + (S == 2 ? (i >> 2) : (i >> 1));
    if (ci < ci_end) {
      int cv;
      const int vi = resolve_view(op, ci, cv);
      const SeistView& v = op.in[vi];
      if (v.g != nullptr && v.bn >= 0) {
        const SeistBN& e = op.bn_table[v.bn];
        atomicAdd(&e.gstat_acc[(i & 1) * e.C + v.bn_c0 + cv], (double)s);
      }
    }
  }
}

// ================================================================================================
// launchers
// ================================================================================================
bool convk_eligible(const SeistOp& op) {
  if (op.pool > 1 || op.n_in != 1) return false;
  if (op.groups > 1 && ((op.Cin / op.groups) < 8 || (op.Cout / op.groups) < 8)) return false;
  if (op.stride != 1 && op.stride != 2) return false;
  switch (op.k) {
    case 3: case 5: case 7: case 9: case 11: case 13: case 15: case 19: break;
    default: return false;
  }
  if (op.stride == 2 && !(op.k == 7 || op.k == 11 || op.k == 15 || op.k == 19)) return false;
  return true;
}

template <typename Kf>
static int ck_set_smem(Kf kernel, size_t bytes) {
  if (bytes > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return (int)e;
  }
  return 0;
}

static int pick_wc(int channels) { return channels > 32 ? 8 : (channels > 16 ? 4 : (channels > 8 ? 2 : 1)); }

// two stages (asynchronous prefetch of the next reduction chunk) where they do not cost a resident CTA below 2 per SM
static int ck_pick_nbuf(size_t bytes1, size_t bytes2) {
  const int knob = env_knob("SEIST_CK_NBUF", 0);
  if (knob == 1 || knob == 2) return bytes2 > 220 * 1024 ? 1 : knob;
  // the second stage costs a resident CTA on most layers of the model family, which loses more than the prefetch wins:
  // two stages only where they are free
  auto ctas = [](size_t b) { return (int)std::min<size_t>(3, (227 * 1024) / (b + 1024)); };
  return (ctas(bytes2) >= ctas(bytes1) && bytes2 <= 220 * 1024) ? 2 : 1;
}

template <int K, int S>
static int launch_fwd_ks(const SeistOp& op, cudaStream_t s) {
  const int gs_out = op.Cout / op.groups;
  const int WC = pick_wc(gs_out), WP = 8 / WC, CO_B = 8 * WC, TLo = 128 * WP;
  const int width = TLo * S + K - S, pitch = ((width + 3) & ~3) + 4;
  const bool up = op.up_src_L > 0;
  const size_t in_f = (size_t)CK_CIC * pitch, w_f = (size_t)CK_CIC * K * CO_B, src_f = up ? (size_t)CK_CIC * (width + 4) : 0;
  auto bytes = [&](int nbuf) { return sizeof(float) * (8 * 16 + (up ? 1 : nbuf) * in_f + nbuf * (w_f + src_f)); };
  const int nbuf = ck_pick_nbuf(bytes(1), bytes(2));
  const size_t smem = bytes(nbuf);
  dim3 grid((op.L_out + TLo - 1) / TLo, op.N, op.groups * ((gs_out + CO_B - 1) / CO_B));
  int rc;
  if (nbuf == 2) {
    rc = ck_set_smem(convk_fwd_kernel<K, S, 2>, smem);
    if (!rc) convk_fwd_kernel<K, S, 2><<<grid, CK_NT, smem, s>>>(op, WC);
  } else {
    rc = ck_set_smem(convk_fwd_kernel<K, S, 1>, smem);
    if (!rc) convk_fwd_kernel<K, S, 1><<<grid, CK_NT, smem, s>>>(op, WC);
  }
  if (rc) return rc;
  note_launch();
  return check_launch("convk_fwd");
}

template <int K, int S>
static int launch_bwdd_k(const SeistOp& op, cudaStream_t s) {
  constexpr int KE = S == 2 ? (K + 1) / 2 : K;
  constexpr int CPW = S == 2 ? 4 : 8;
  const int gs_in = op.Cin / op.groups;
  const int WC = pick_wc(gs_in * (8 / CPW)), WP = 8 / WC, CI_B = CPW * WC, TLo = 128 * WP;
  const int width = TLo + KE - 1, pitch = ((width + 3) & ~3) + 4;
  const bool has_bn = op.out.bn >= 0 && op.out.g != nullptr;
  const bool need_x = has_bn || op.out_act == SEIST_OUT_SIGMOID;
  const int nraw = !need_x ? 1 : ((has_bn && op.out_dxd != nullptr) ? 3 : 2);
  const size_t z_f = (size_t)CK_CIC * pitch, w_f = (size_t)CK_CIC * KE * 8 * WC;
  auto bytes = [&](int nbuf) { return sizeof(float) * (8 * 16 + nbuf * (nraw * z_f + w_f)); };
  const int nbuf = ck_pick_nbuf(bytes(1), bytes(2));
  const size_t smem = bytes(nbuf);
  dim3 grid(((op.L_in + S - 1) / S + TLo - 1) / TLo, op.N, op.groups * ((gs_in + CI_B - 1) / CI_B));
  int rc;
  if (nbuf == 2) {
    rc = ck_set_smem(convk_bwd_data_kernel<K, S, 2>, smem);
    if (!rc) convk_bwd_data_kernel<K, S, 2><<<grid, CK_NT, smem, s>>>(op, WC, nraw);
  } else {
    rc = ck_set_smem(convk_bwd_data_kernel<K, S, 1>, smem);
    if (!rc) convk_bwd_data_kernel<K, S, 1><<<grid, CK_NT, smem, s>>>(op, WC, nraw);
  }
  if (rc) return rc;
  note_launch();
  return check_launch("convk_bwd_data");
}

#define CK_SWITCH_K(FN, ...)              \
  switch (op.k) {                         \
    case 3: return FN(3, __VA_ARGS__);    \
    case 5: return FN(5, __VA_ARGS__);    \
    case 7: return FN(7, __VA_ARGS__);    \
    case 9: return FN(9, __VA_ARGS__);    \
    case 11: return FN(11, __VA_ARGS__);  \
    case 13: return FN(13, __VA_ARGS__);  \
    case 15: return FN(15, __VA_ARGS__);  \
    default: return FN(19, __VA_ARGS__);  \
  }

int launch_convk_fwd(const SeistOp& op, cudaStream_t s) {
  if (op.stride == 2) {
    switch (op.k) {
      case 7: return launch_fwd_ks<7, 2>(op, s);
      case 11: return launch_fwd_ks<11, 2>(op, s);
      case 15: return launch_fwd_ks<15, 2>(op, s);
      default: return launch_fwd_ks<19, 2>(op, s);
    }
  }
#define FWD1(KK, dummy) launch_fwd_ks<KK, 1>(op, s)
  CK_SWITCH_K(FWD1, 0)
#undef FWD1
}

// stride 2 needs an even left pad and no up-sampling (true for every strided conv of the model family)
bool convk_bwd_data_eligible(const SeistOp& op) {
  if (!convk_eligible(op)) return false;
  if (op.stride == 1) return true;
  return (op.pad_left & 1) == 0 && op.up_src_L == 0;
}

int launch_convk_bwd_data(const SeistOp& op, cudaStream_t s) {
  if (op.stride == 2) {
    switch (op.k) {
      case 7: return launch_bwdd_k<7, 2>(op, s);
      case 11: return launch_bwdd_k<11, 2>(op, s);
      case 15: return launch_bwdd_k<15, 2>(op, s);
      default: return launch_bwdd_k<19, 2>(op, s);
    }
  }
#define BD(KK, dummy) launch_bwdd_k<KK, 1>(op, s)
  CK_SWITCH_K(BD, 0)
#undef BD
}

}  // namespace seist
