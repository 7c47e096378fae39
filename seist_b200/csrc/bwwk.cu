// Weight gradient of the dense k-tap convolutions (k > 1): composed stem paths, MSMC branches, the dpk head
// (reference models/seist.py:86-111 stem, :225-287 MSMC, :566-575 head up-sampling + conv).
//
//   dW[co][ci][t] = sum_{n,l} gacc[co][n,l] * convin[ci][n, l*S + t - pad_left]
//
// Sliding-window formulation: a thread owns 4 output channels x ONE input channel x all K taps.  For a quad
// of 4 consecutive output samples it reads the 4 gacc quads (broadcast across the lanes that share the
// channel group) and the K+3S input samples the quad touches as ceil((K+3S)/4) 16-byte shared loads, then
// issues 16*K FMAs - the taps of one input channel re-use the same window out of registers instead of
// re-reading it once per tap as the row-tiled kernel in pw.cu does (k = 7: 112 FMA per 7 LDS.128).
//
// A CTA owns a (4*TGM) x CI_B tile of (co, ci) pairs and a strided share of the PC-sample chunks of all
// waveforms.  Per chunk every gacc / input element is loaded and transformed ONCE into shared memory
// (BN-backward prologue for gacc; BN-apply / GELU / up-sampling / zero padding for the input).  Threads are
// laid out as TG = TGM*nci tile coordinates x PG sample groups; the sample groups are folded through shared
// memory at the end, one float atomic per dW element per CTA.
//
// fma2: the gacc rows are parked in shared memory interleaved in channel pairs ({g[2r][s], g[2r+1][s]}), so a
// 16-byte load yields two aligned (even, odd channel) register pairs; each fma2 multiplies such a pair with one
// broadcast window sample: 8*K packed FMAs per quad instead of 16*K scalar ones.
#include <algorithm>
#include "common.cuh"
#include "conv_common.cuh"

namespace seist {

constexpr int BK_NT = 256;

namespace {
__device__ __forceinline__ float4 bk_ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 bk_ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void bk_st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
struct BkOut {
  float A, Bx, Cc, pad;
};
}  // namespace

template <int K, int S, int TGM, int NPR>   // NPR pair rows (2*NPR output channels) per thread
__global__ void __launch_bounds__(BK_NT, (K <= 9 && NPR == 2) ? 3 : 2) bwwk_kernel(const __grid_constant__ SeistOp op, const int CI_B, const int PC,
                                                        const int pitch, const int area_f, const int gx_off) {
  constexpr int CO_B = 2 * NPR * TGM;
  constexpr int WN = K + 3 * S, WQ = (WN + 3) / 4;
  constexpr int RW = (K + 1) | 1;                      // odd row pitch of the final fold
  extern __shared__ __align__(16) unsigned char sm_raw[];
  const int L = op.L_out;
  const int gpitch = 2 * PC + 8;                         // pitch of a channel-PAIR row (= 8 mod 32 floats)
  const int gs_in = op.Cin / op.groups, gs_out = op.Cout / op.groups;
  const int tpg = (gs_out + CO_B - 1) / CO_B;            // output-channel tiles per group
  const int grp = blockIdx.y / tpg;
  const int Cin_hi = (grp + 1) * gs_in, Cout_hi = (grp + 1) * gs_out;
  const int width = PC * S + K - S;
  float* g_s = reinterpret_cast<float*>(sm_raw);          // [CO_B/2][gpitch]
  float* in_s = g_s + (CO_B / 2) * gpitch;                // [CI_B][pitch]
  BkOut* oc_s = reinterpret_cast<BkOut*>(g_s + area_f);   // [CO_B]
  float* src_s = reinterpret_cast<float*>(oc_s + CO_B);   // [CI_B][width+4] (up-sampled input only)
  float* gx_s = reinterpret_cast<float*>(sm_raw) + (gx_off > 0 ? gx_off : 0);   // raw x / dxd planes of the asynchronous gacc staging
  float* gd_s = gx_s + (CO_B / 2) * gpitch;
  const int tid = threadIdx.x;
  const int co_base = grp * gs_out + (blockIdx.y - grp * tpg) * CO_B;
  const int ci_lo = grp * gs_in + blockIdx.z * CI_B;
  const int nci = min(CI_B, Cin_hi - ci_lo);

  for (int col = tid; col < CO_B; col += BK_NT) {
    const int co = co_base + col;
    BkOut o = {0.f, 0.f, 0.f, 0.f};
    if (co < Cout_hi) {
      const OutGradCoef kc = out_grad_coef(op, co);
      o.A = kc.A;
      o.Bx = kc.Bx;
      o.Cc = kc.Cc;
    }
    oc_s[col] = o;
  }
  __syncthreads();

  const uint64_t seed = load_seed(op.step_seed);
  const bool has_bn = (op.out.bn >= 0 && op.out.g != nullptr);
  const bool need_x = has_bn || op.out_act == SEIST_OUT_SIGMOID;
  const int Lsrc = op.in[0].L;
  const float ratio = op.up_src_L > 0 ? (float)Lsrc / (float)op.L_in : 1.f;
  const int TG = TGM * nci, PG = BK_NT / TG;
  const int tcoord = tid % TG, pg = tid / TG;
  const bool active = pg < PG;
  const int tm = tcoord / nci, tn = tcoord - tm * nci;
  const float* my_in = in_s + tn * pitch;
  const float* my_g = g_s + tm * gpitch;                  // pair rows tm + TGM*ip: channels 2*(tm + TGM*ip) + {0,1}

  float2 acc[NPR][K];                                     // [pair row ip][tap]: .x even channel, .y odd channel
  float2 bacc[NPR];
#pragma unroll
  for (int i = 0; i < NPR; ++i) {
    bacc[i] = make_float2(0.f, 0.f);
#pragma unroll
    for (int t = 0; t < K; ++t) acc[i][t] = make_float2(0.f, 0.f);
  }

  const int chunks_per_n = (L + PC - 1) / PC;
  const int total = op.N * chunks_per_n;
  const int QPR = PC >> 2;
  for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
    const int n = tile / chunks_per_n;
    const int l0 = (tile - n * chunks_per_n) * PC;
    const float pf = path_factor(op, seed, n) * alpha_factor(op, seed, n);
    // ---- conv-input rows: in_s[r][pos] <-> conv-input coordinate p_base + pos.  Plain rows are copied raw and
    // asynchronously FIRST (their latency hides behind the gacc loads) and transformed in place below
    const int p_base = l0 * S - op.pad_left;
    if (op.up_src_L == 0) {
      rows_issue_plain(op, n, ci_lo, nci, nci, in_s, pitch, width, p_base);
      cp_async_commit();
    }
    // ---- gacc rows, interleaved in channel pairs: g_s[pr][2*s + half] ---------------------------------
    if (gx_off > 0) {
      gacc_issue<BK_NT>(op, n, l0, L, co_base, Cout_hi, CO_B, QPR, gpitch, g_s, gx_s, gd_s, has_bn, need_x);
      cp_async_commit();
      cp_async_wait<0>();
      gacc_combine<BK_NT>(op, n, l0, L, co_base, Cout_hi, CO_B, QPR, gpitch, g_s, gx_s, gd_s, oc_s, has_bn, need_x, pf, seed, op.Cout);
    } else
    for (int idx = tid; idx < (CO_B / 2) * QPR; idx += BK_NT) {
      const int pr = idx / QPR, q = idx - pr * QPR;
      const int l = l0 + 4 * q;
      float4 gh[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = 2 * pr + h, co = co_base + row;
        float4 gv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (co < Cout_hi && l < L) {
          const size_t off = ((size_t)n * op.out.Ct + op.out.c0 + co) * (size_t)L + l;
          if (op.out_dxd) gv = bk_ldg4(op.out_dxd + off);
          if (need_x) {
            const float4 x = bk_ldg4(op.out.x + off);
            if (has_bn) {
              const float4 du = bk_ldg4(op.out.g + off);
              const BkOut o = oc_s[row];
              gv = add4(gv, fma4(splat4(o.A), du, fma4(splat4(o.Bx), x, splat4(o.Cc))));
            }
            if (op.out_act == SEIST_OUT_SIGMOID) gv = mul4(gv, mul4(x, fma4(x, splat4(-1.f), splat4(1.f))));
          }
          gv = scale4(gv, pf);
          if (op.p_elem > 0.f) gv = mul4(gv, keep4(op.p_elem, seed, op.seed_elem, ((uint64_t)n * op.Cout + co) * (uint64_t)L + l));
        }
        gh[h] = gv;
      }
      float* gp = g_s + pr * gpitch + 8 * q;
      bk_st4(gp, make_float4(gh[0].x, gh[1].x, gh[0].y, gh[1].y));
      bk_st4(gp + 4, make_float4(gh[0].z, gh[1].z, gh[0].w, gh[1].w));
    }
    if (op.up_src_L > 0) {
      stage_upsampled_rows(op, n, ci_lo, nci, in_s, pitch, width, p_base, src_s, width + 4, Lsrc, ratio);
    } else {
      cp_async_wait<0>();
      rows_transform_plain(op, n, ci_lo, nci, in_s, pitch, width, p_base);
    }
    __syncthreads();
    // ---- accumulate -------------------------------------------------------------------------------
    if (active) {
      for (int q = pg; q < QPR; q += PG) {
        float w[4 * WQ];
        const float* ip = my_in + 4 * q * S;
#pragma unroll
        for (int j = 0; j < WQ; ++j) {
          const float4 t4 = bk_ld4(ip + 4 * j);
          w[4 * j] = t4.x;
          w[4 * j + 1] = t4.y;
          w[4 * j + 2] = t4.z;
          w[4 * j + 3] = t4.w;
        }
        float2 gp[NPR][4];                                // [pair row][sample]
#pragma unroll
        for (int i = 0; i < NPR; ++i) {
          const float4 a = bk_ld4(my_g + TGM * i * gpitch + 8 * q), b = bk_ld4(my_g + TGM * i * gpitch + 8 * q + 4);
          gp[i][0] = make_float2(a.x, a.y);
          gp[i][1] = make_float2(a.z, a.w);
          gp[i][2] = make_float2(b.x, b.y);
          gp[i][3] = make_float2(b.z, b.w);
        }
#pragma unroll
        for (int t = 0; t < K; ++t) {
#pragma unroll
          for (int i = 0; i < NPR; ++i) {
            float2 a = acc[i][t];
            a = fma2(gp[i][0], dup2(w[t]), a);
            a = fma2(gp[i][1], dup2(w[S + t]), a);
            a = fma2(gp[i][2], dup2(w[2 * S + t]), a);
            a = fma2(gp[i][3], dup2(w[3 * S + t]), a);
            acc[i][t] = a;
          }
        }
        if (tn == 0) {
#pragma unroll
          for (int i = 0; i < NPR; ++i) {
            bacc[i].x += (gp[i][0].x + gp[i][1].x) + (gp[i][2].x + gp[i][3].x);
            bacc[i].y += (gp[i][0].y + gp[i][1].y) + (gp[i][2].y + gp[i][3].y);
          }
        }
      }
    }
    __syncthreads();
  }

  // ---- fold the sample groups through shared memory, one channel group (i) per round --------------------
  float* red = g_s;
  const int R = gs_in * K;
#pragma unroll
  for (int i = 0; i < 2 * NPR; ++i) {                     // round i: pair row ip = i >> 1, half = i & 1
    float* mine = red + (size_t)tid * RW;
#pragma unroll
    for (int t = 0; t < K; ++t) mine[t] = (i & 1) ? acc[i >> 1][t].y : acc[i >> 1][t].x;
    mine[K] = (i & 1) ? bacc[i >> 1].y : bacc[i >> 1].x;
    __syncthreads();
    for (int idx = tid; idx < TG * (K + 1); idx += BK_NT) {
      const int tc = idx / (K + 1), e = idx - tc * (K + 1);
      float s = 0.f;
      for (int p = 0; p < PG; ++p) s += red[((size_t)p * TG + tc) * RW + e];
      const int m = tc / nci, cr = tc - m * nci;
      const int co = co_base + 2 * (m + TGM * (i >> 1)) + (i & 1);
      if (co < Cout_hi) {
        if (e < K) {
          atomicAdd(&op.dW[(size_t)co * R + (size_t)(ci_lo - grp * gs_in + cr) * K + e], s);
        } else if (cr == 0 && blockIdx.z == 0 && op.dbias != nullptr) {
          atomicAdd(&op.dbias[co], s);
        }
      }
    }
    __syncthreads();
  }
}

template <int K, int S, int TGM, int NPR>
static int launch_bwwk_t(const SeistOp& op, cudaStream_t s, int sm_count) {
  constexpr int CO_B = 2 * NPR * TGM;
  constexpr int WQ = (K + 3 * S + 3) / 4;
  constexpr int RW = (K + 1) | 1;
  const int gs_in = op.Cin / op.groups, gs_out = op.Cout / op.groups;
  const int ntile = (gs_in + 15) / 16;
  const int CI_B = (gs_in + ntile - 1) / ntile;          // balanced input-channel tiles of at most 16
  int PC = 128;
  if (op.L_out >= 2048 && CO_B + CI_B <= 24) PC = 512;
  else if (op.L_out >= 256) PC = 256;
  if (PC > ((op.L_out + 3) & ~3)) PC = (op.L_out + 3) & ~3;
  const int width = PC * S + K - S;
  // row pitch: room for the last quad's window over-read, 16-byte aligned, = 4 (mod 32) so that the 8 lanes
  // of a quarter warp reading 8 different rows hit 8 different 16-byte bank groups
  int pitch = (4 * (PC / 4 - 1) * S + 4 * WQ + 3) & ~3;
  if (pitch < ((width + 3) & ~3)) pitch = (width + 3) & ~3;
  while ((pitch & 31) != 4) pitch += 4;
  int area_f = (CO_B / 2) * (2 * PC + 8) + CI_B * pitch;
  if (area_f < BK_NT * RW) area_f = BK_NT * RW;
  area_f = (area_f + 3) & ~3;
  size_t smem = sizeof(float) * (size_t)area_f + sizeof(BkOut) * CO_B +
                (op.up_src_L > 0 ? sizeof(float) * (size_t)CI_B * (width + 4) : 0) + 16;
  // raw planes of the asynchronous gacc staging (x, dxd next to du) - unless they would cost a resident CTA
  int gx_off = 0;
  if (env_knob("SEIST_ASYNC", 7) & 8) {   // opt-in: it helps the row-tiled kernel more than this one
    const bool has_bn = op.out.bn >= 0 && op.out.g != nullptr;
    const bool need_x = has_bn || op.out_act == SEIST_OUT_SIGMOID;
    const int planes = (need_x ? 1 : 0) + ((has_bn && op.out_dxd != nullptr) ? 1 : 0);
    const size_t base = (smem + 15) & ~(size_t)15;
    const size_t extra = sizeof(float) * (size_t)planes * (CO_B / 2) * (2 * PC + 8);
    auto ctas = [](size_t b) { return (227 * 1024) / (b + 1024); };
    const size_t cap = (K <= 9 && NPR == 2) ? 3 : 2;      // __launch_bounds__ of the kernel
    if (std::min(cap, ctas(base + extra)) >= std::min(cap, ctas(base))) {
      gx_off = (int)(base / sizeof(float));
      smem = base + extra;
    }
  }
  const int gy = op.groups * ((gs_out + CO_B - 1) / CO_B), gz = ntile;
  const long tiles = (long)op.N * ((op.L_out + PC - 1) / PC);
  long gx = ((long)bww_waves() * sm_count + gy * gz - 1) / (gy * gz);
  if (gx > tiles) gx = tiles;
  if (gx < 1) gx = 1;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(bwwk_kernel<K, S, TGM, NPR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
  }
  bwwk_kernel<K, S, TGM, NPR><<<dim3((unsigned)gx, gy, gz), BK_NT, smem, s>>>(op, CI_B, PC, pitch, area_f, gx_off);
  note_launch();
  return check_launch("bwwk");
}

template <int K, int S>
static int launch_bwwk_ks(const SeistOp& op, cudaStream_t s, int sm_count) {
  if (op.Cout / op.groups <= 8) return launch_bwwk_t<K, S, 2, 2>(op, s, sm_count);
  // wide output tiles (32 channels, 8 per thread) halve the re-staging of the input rows; the 4*K extra
  // accumulator registers fit for the short filters only
  if constexpr (K <= 7 && S == 1) {
    if (op.Cout / op.groups >= 32) return launch_bwwk_t<K, S, 4, 4>(op, s, sm_count);
  }
  return launch_bwwk_t<K, S, 4, 2>(op, s, sm_count);
}

static bool bwwk_has(int k, int stride) {
  if (stride == 1) return k == 3 || k == 5 || k == 7 || k == 9 || k == 11 || k == 13;
  if (stride == 2) return k == 7 || k == 11 || k == 15 || k == 19;
  return false;
}

// eligibility: one input view, no pooling, whole quads, a compiled (k, stride) pair
bool bwwk_eligible(const SeistOp& op) {
  if (op.n_in != 1 || op.pool > 1 || (op.L_out & 3)) return false;
  if (op.Cin % op.groups || op.Cout % op.groups) return false;
  return bwwk_has(op.k, op.stride);
}

int launch_bwwk(const SeistOp& op, cudaStream_t s, int sm_count) {
  if (op.stride == 1) {
    switch (op.k) {
      case 3: return launch_bwwk_ks<3, 1>(op, s, sm_count);
      case 5: return launch_bwwk_ks<5, 1>(op, s, sm_count);
      case 7: return launch_bwwk_ks<7, 1>(op, s, sm_count);
      case 9: return launch_bwwk_ks<9, 1>(op, s, sm_count);
      case 11: return launch_bwwk_ks<11, 1>(op, s, sm_count);
      case 13: return launch_bwwk_ks<13, 1>(op, s, sm_count);
    }
  } else if (op.stride == 2) {
    switch (op.k) {
      case 7: return launch_bwwk_ks<7, 2>(op, s, sm_count);
      case 11: return launch_bwwk_ks<11, 2>(op, s, sm_count);
      case 15: return launch_bwwk_ks<15, 2>(op, s, sm_count);
      case 19: return launch_bwwk_ks<19, 2>(op, s, sm_count);
    }
  }
  set_error("bwwk: no kernel compiled for this (k, stride)");
  return -1;
}

}  // namespace seist
