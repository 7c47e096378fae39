// Small kernels: regression/classification head, BatchNorm finalisation, fused losses, fused Adam and SGD.
#include "common.cuh"

namespace seist {

// ================================================================================================
// HeadRegression / HeadClassification (reference models/seist.py:575-610):
//   y = act( W . mean_L(x) + b ),  act = sigmoid * scale | softmax
// grid N, 128 threads.  Shared: mean[C], z[nout].
// ================================================================================================
__device__ __forceinline__ void headvec_mean(const SeistOp& op, int n, float* mean_s) {
  const SeistView& v = op.in[0];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int c = warp; c < v.C; c += 4) {
    float sc, sh;
    view_coef(op, v, c, sc, sh);
    const float* xr = view_row(v, n, c);
    float s = 0.f;
    for (int l = lane; l < v.L; l += 32) {
      const float u = fmaf(sc, xr[l], sh);
      s += v.act == SEIST_ACT_GELU ? gelu_f(u) : u;
    }
    s = warp_sum(s);
    if (lane == 0) mean_s[c] = s / (float)v.L;
  }
}

__global__ void __launch_bounds__(128) headvec_fwd_kernel(const __grid_constant__ SeistOp op) {
  extern __shared__ float sm[];
  float* mean_s = sm;
  float* z_s = sm + op.Cin;
  const int n = blockIdx.x;
  headvec_mean(op, n, mean_s);
  __syncthreads();
  for (int o = threadIdx.x; o < op.Cout; o += blockDim.x) {
    float z = op.bias ? op.bias[o] : 0.f;
    for (int c = 0; c < op.Cin; ++c) z = fmaf(op.W[o * op.Cin + c], mean_s[c], z);
    z_s[o] = z;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float* y = op.out.x + (size_t)n * op.Cout;
    if (op.out_act == SEIST_OUT_SIGMOID) {
      for (int o = 0; o < op.Cout; ++o) y[o] = op.out_scale / (1.f + expf(-z_s[o]));
    } else if (op.out_act == SEIST_OUT_SOFTMAX) {
      float m = -INFINITY, d = 0.f;
      for (int o = 0; o < op.Cout; ++o) m = fmaxf(m, z_s[o]);
      for (int o = 0; o < op.Cout; ++o) d += expf(z_s[o] - m);
      for (int o = 0; o < op.Cout; ++o) y[o] = expf(z_s[o] - m) / d;
    } else {
      for (int o = 0; o < op.Cout; ++o) y[o] = z_s[o];
    }
  }
}

__global__ void __launch_bounds__(128) headvec_bwd_kernel(const __grid_constant__ SeistOp op) {
  extern __shared__ float sm[];
  float* mean_s = sm;
  float* dz_s = sm + op.Cin;
  const int n = blockIdx.x;
  headvec_mean(op, n, mean_s);
  if (threadIdx.x == 0) {
    const float* y = op.out.x + (size_t)n * op.Cout;
    const float* dy = op.out_dxd + (size_t)n * op.Cout;
    if (op.out_act == SEIST_OUT_SIGMOID) {
      for (int o = 0; o < op.Cout; ++o) {
        const float sg = y[o] / op.out_scale;
        dz_s[o] = dy[o] * op.out_scale * sg * (1.f - sg);
      }
    } else if (op.out_act == SEIST_OUT_SOFTMAX) {
      float dot = 0.f;
      for (int o = 0; o < op.Cout; ++o) dot += y[o] * dy[o];
      for (int o = 0; o < op.Cout; ++o) dz_s[o] = y[o] * (dy[o] - dot);
    } else {
      for (int o = 0; o < op.Cout; ++o) dz_s[o] = dy[o];
    }
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < op.Cout * op.Cin; idx += blockDim.x) {
    const int o = idx / op.Cin, c = idx - o * op.Cin;
    atomicAdd(&op.dW[idx], dz_s[o] * mean_s[c]);
  }
  if (op.dbias != nullptr)
    for (int o = threadIdx.x; o < op.Cout; o += blockDim.x) atomicAdd(&op.dbias[o], dz_s[o]);
  const SeistView& v = op.in[0];
  if (v.g == nullptr) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int c = warp; c < v.C; c += 4) {
    float dm = 0.f;
    for (int o = 0; o < op.Cout; ++o) dm = fmaf(op.W[o * op.Cin + c], dz_s[o], dm);
    dm /= (float)v.L;
    float sc, sh, mu = 0.f, istd = 0.f;
    view_coef(op, v, c, sc, sh);
    if (v.bn >= 0) view_khat(op, v, c, mu, istd);
    const float* xr = view_row(v, n, c);
    float* gr = view_grad_row(v, n, c);
    float s1 = 0.f, s2 = 0.f;
    for (int l = lane; l < v.L; l += 32) {
      const float x = xr[l];
      float g = dm;
      if (v.act == SEIST_ACT_GELU) g *= gelu_grad_f(fmaf(sc, x, sh));
      if (v.accum) gr[l] += g; else gr[l] = g;
      s1 += g;
      s2 = fmaf(g, (x - mu) * istd, s2);
    }
    if (v.bn >= 0) {
      s1 = warp_sum(s1);
      s2 = warp_sum(s2);
      if (lane == 0) gstat_add(op, v, c, s1, s2);
    }
  }
}

int launch_headvec_fwd(const SeistOp& op, cudaStream_t s) {
  headvec_fwd_kernel<<<op.N, 128, sizeof(float) * (op.Cin + op.Cout), s>>>(op);
  note_launch();
  return check_launch("headvec_fwd");
}
int launch_headvec_bwd(const SeistOp& op, cudaStream_t s) {
  headvec_bwd_kernel<<<op.N, 128, sizeof(float) * (op.Cin + op.Cout), s>>>(op);
  note_launch();
  return check_launch("headvec_bwd");
}

// ================================================================================================
// BatchNorm finalisation: one block per BN entry.
// ================================================================================================
__global__ void bn_finalize_fwd_kernel(const SeistBN* tab, int n_bn) {
  const SeistBN& e = tab[blockIdx.x];
  if (!e.use_batch || e.is_chained) return;
  const double unb = e.count > 1.0 ? e.count / (e.count - 1.0) : 1.0;
  for (int c = threadIdx.x; c < e.C; c += blockDim.x) {
    double mean, var;
    bn_moments(e, c, mean, var);
    const double mom = e.momentum;
    e.running_mean[c] = (float)((1.0 - mom) * (double)e.running_mean[c] + mom * mean);
    e.running_var[c] = (float)((1.0 - mom) * (double)e.running_var[c] + mom * var * unb);
    if (e.chain >= 0) {
      const SeistBN& e2 = tab[e.chain];
      const double g1 = e.gamma[c], b1 = e.beta[c];
      const double var2 = g1 * g1 * var / (var + (double)e.eps);
      const double m2 = e2.momentum;
      e2.running_mean[c] = (float)((1.0 - m2) * (double)e2.running_mean[c] + m2 * b1);
      e2.running_var[c] = (float)((1.0 - m2) * (double)e2.running_var[c] + m2 * var2 * unb);
    }
  }
}

__global__ void bn_finalize_bwd_kernel(const SeistBN* tab, int n_bn) {
  const SeistBN& e = tab[blockIdx.x];
  if (!e.use_batch || e.is_chained) return;
  for (int c = threadIdx.x; c < e.C; c += blockDim.x) {
    const double S1 = e.gstat[c], S2 = e.gstat[e.C + c];
    const double gs = e.grad_scale;
    if (e.chain < 0) {
      e.dgamma[c] += (float)(S2 * gs);
      e.dbeta[c] += (float)(S1 * gs);
    } else {
      const SeistBN& e2 = tab[e.chain];
      double mean, var;
      bn_moments(e, c, mean, var);
      const double istd = rsqrt(var + (double)e.eps);
      const double g1 = e.gamma[c], g2 = e2.gamma[c];
      const double vk = var * istd * istd;
      const double istd2 = rsqrt(g1 * g1 * vk + (double)e2.eps);
      e2.dbeta[c] += (float)(S1 * gs);
      e2.dgamma[c] += (float)(g1 * istd2 * S2 * gs);
      e.dgamma[c] += (float)(g2 * istd2 * S2 * (1.0 - g1 * g1 * istd2 * istd2 * vk) * gs);
      // d(beta) of the first BN of a chain is analytically zero
    }
  }
}

// per-channel coefficient tables (see SeistBN::coef): one block per BN entry of [bn_lo, bn_lo + n)
__global__ void bn_prepare_fwd_kernel(const SeistBN* tab, int bn_lo) {
  const int bn = bn_lo + blockIdx.x;
  const SeistBN& e = tab[bn];
  if (e.is_chained) return;
  for (int c = threadIdx.x; c < e.C; c += blockDim.x) {
    float* k = e.coef + 8 * (size_t)c;
    bn_fwd_coef(tab, bn, c, k[0], k[1]);
    bn_khat_coef(tab, bn, c, k[2], k[3]);
  }
}
__global__ void bn_prepare_bwd_kernel(const SeistBN* tab, int bn_lo) {
  const int bn = bn_lo + blockIdx.x;
  const SeistBN& e = tab[bn];
  if (e.is_chained) return;
  for (int c = threadIdx.x; c < e.C; c += blockDim.x) {
    float* k = e.coef + 8 * (size_t)c;
    bn_bwd_coef(tab, bn, c, k[4], k[5], k[6]);
  }
}
int launch_bn_prepare_xchg(const SeistOp& op, bool fwd, cudaStream_t s);
int launch_bn_prepare(const SeistOp& op, bool fwd, cudaStream_t s) {
  if (op.n_bn <= 0) return 0;
  if (op.comm != nullptr) return launch_bn_prepare_xchg(op, fwd, s);     // data parallel: statistic sum over peer memory fused in
  if (fwd) bn_prepare_fwd_kernel<<<op.n_bn, 64, 0, s>>>(op.bn_table, op.bn_lo);
  else bn_prepare_bwd_kernel<<<op.n_bn, 64, 0, s>>>(op.bn_table, op.bn_lo);
  note_launch();
  return check_launch("bn_prepare");
}

// ---- stem path weight composition (SEIST_OP_STEM_COMPOSE_*) -----------------------------------------
__global__ void stem_compose_fwd_kernel(const float* __restrict__ I, const float* __restrict__ D,
                                        const float* __restrict__ P, float* __restrict__ We, int C, int Cout, int k) {
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < Cout * C * k; idx += gridDim.x * blockDim.x) {
    const int t = idx % k, i = (idx / k) % C, o = idx / (k * C);
    float s = 0.f;
    for (int c = 0; c < C; ++c) s = fmaf(P[o * C + c] * D[c * k + t], I[c * C + i], s);
    We[idx] = s;
  }
}
__global__ void stem_compose_bwd_kernel(const float* __restrict__ I, const float* __restrict__ D,
                                        const float* __restrict__ P, const float* __restrict__ dWe, float* dI,
                                        float* dD, float* dP, int C, int Cout, int k) {
  const int nI = C * C, nD = C * k, nP = Cout * C;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < nI + nD + nP; idx += gridDim.x * blockDim.x) {
    float s = 0.f;
    if (idx < nI) {                       // dI[c][i] = sum_{o,t} dWe[o][i][t] P[o][c] D[c][t]
      const int c = idx / C, i = idx % C;
      for (int o = 0; o < Cout; ++o)
        for (int t = 0; t < k; ++t) s = fmaf(dWe[(o * C + i) * k + t] * P[o * C + c], D[c * k + t], s);
      dI[idx] += s;
    } else if (idx < nI + nD) {           // dD[c][t] = sum_{o,i} dWe[o][i][t] P[o][c] I[c][i]
      const int j = idx - nI, c = j / k, t = j % k;
      for (int o = 0; o < Cout; ++o)
        for (int i = 0; i < C; ++i) s = fmaf(dWe[(o * C + i) * k + t] * P[o * C + c], I[c * C + i], s);
      dD[j] += s;
    } else {                              // dP[o][c] = sum_{i,t} dWe[o][i][t] D[c][t] I[c][i]
      const int j = idx - nI - nD, o = j / C, c = j % C;
      for (int i = 0; i < C; ++i)
        for (int t = 0; t < k; ++t) s = fmaf(dWe[(o * C + i) * k + t] * D[c * k + t], I[c * C + i], s);
      dP[j] += s;
    }
  }
}
int launch_stem_compose(const SeistOp& op, bool fwd, cudaStream_t s) {
  const int C = op.Cin, Cout = op.Cout, k = op.k;
  if (fwd) {
    stem_compose_fwd_kernel<<<(Cout * C * k + 255) / 256, 256, 0, s>>>(op.in[0].x, op.in[1].x, op.in[2].x, op.out.x, C,
                                                                       Cout, k);
  } else {
    stem_compose_bwd_kernel<<<(C * C + C * k + Cout * C + 127) / 128, 128, 0, s>>>(
        op.in[0].x, op.in[1].x, op.in[2].x, op.out.g, op.in[0].g, op.in[1].g, op.in[2].g, C, Cout, k);
  }
  note_launch();
  return check_launch("stem_compose");
}

int launch_bn_finalize(const SeistOp& op, bool fwd, cudaStream_t s) {
  if (op.n_bn <= 0) return 0;
  if (fwd) bn_finalize_fwd_kernel<<<op.n_bn, 64, 0, s>>>(op.bn_table, op.n_bn);
  else bn_finalize_bwd_kernel<<<op.n_bn, 64, 0, s>>>(op.bn_table, op.n_bn);
  note_launch();
  return check_launch("bn_finalize");
}

// ================================================================================================
// losses
// ================================================================================================
__device__ __forceinline__ float block_sum_128(float v) {
  __shared__ float part[8];
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) part[warp] = v;
  __syncthreads();
  float t = 0.f;
  if (warp == 0) {
    t = lane < (int)(blockDim.x >> 5) ? part[lane] : 0.f;
    t = warp_sum(t);
  }
  return t;   // valid in thread 0
}

__global__ void __launch_bounds__(256) bce_fwd_kernel(const float* __restrict__ p, const float* __restrict__ t,
                                                      const float* __restrict__ w, int64_t total, int C, int64_t L,
                                                      float eps, double* acc) {
  float s = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)((i / L) % C);
    const float pi = p[i], ti = t[i];
    s -= w[c] * (ti * logf(pi + eps) + (1.f - ti) * logf(1.f - pi + eps));
  }
  s = block_sum_128(s);
  if (threadIdx.x == 0) atomicAdd(acc, (double)s);
}

__global__ void mean_finalize_kernel(const double* acc, double inv, float* out) { *out = (float)(*acc * inv); }

__global__ void __launch_bounds__(256) bce_bwd_kernel(const float* __restrict__ p, const float* __restrict__ t,
                                                      const float* __restrict__ w, const float* __restrict__ gout,
                                                      int64_t total, int C, int64_t L, float eps, float inv,
                                                      float* __restrict__ d) {
  const float go = gout[0] * inv;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)((i / L) % C);
    const float pi = p[i], ti = t[i];
    d[i] = -go * w[c] * (ti / (pi + eps) - (1.f - ti) / (1.f - pi + eps));
  }
}

__global__ void __launch_bounds__(256) huber_fwd_kernel(const float* __restrict__ p, const float* __restrict__ t,
                                                        int64_t total, float delta, double* acc) {
  float s = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const float d = fabsf(p[i] - t[i]);
    s += d <= delta ? 0.5f * d * d : delta * (d - 0.5f * delta);
  }
  s = block_sum_128(s);
  if (threadIdx.x == 0) atomicAdd(acc, (double)s);
}

__global__ void __launch_bounds__(256) huber_bwd_kernel(const float* __restrict__ p, const float* __restrict__ t,
                                                        const float* __restrict__ gout, int64_t total, float delta,
                                                        float inv, float* __restrict__ d) {
  const float go = gout[0] * inv;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const float r = p[i] - t[i];
    d[i] = go * (fabsf(r) <= delta ? r : (r > 0.f ? delta : -delta));
  }
}

// CELoss (reference models/loss.py:8-29): mean over rows of sum_c -w[c] * t[c] * log(p[c] + eps); preds are probabilities
// (the classification head ends in a softmax, models/seist.py:575-591)
__global__ void __launch_bounds__(256) ce_fwd_kernel(const float* __restrict__ p, const float* __restrict__ t,
                                                     const float* __restrict__ w, int64_t total, int C, float eps, double* acc) {
  float s = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    s -= w[i % C] * t[i] * logf(p[i] + eps);
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0 && s != 0.f) atomicAdd(acc, (double)s);
}
__global__ void __launch_bounds__(256) ce_bwd_kernel(const float* __restrict__ p, const float* __restrict__ t,
                                                     const float* __restrict__ w, const float* __restrict__ gout, int64_t total,
                                                     int C, float eps, float inv_rows, float* __restrict__ d) {
  const float g = *gout * inv_rows;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    d[i] = -g * w[i % C] * t[i] / (p[i] + eps);
}

static int ew_grid(int64_t total) {
  int64_t g = (total + 256 * 8 - 1) / (256 * 8);
  if (g < 1) g = 1;
  if (g > 132 * 16) g = 132 * 16;
  return (int)g;
}

// ================================================================================================
// Adam
// ================================================================================================
// torch.optim.Adam's arithmetic: hyper-parameters are python doubles there, so (1 - beta) and the bias corrections are
// formed in double before rounding to fp32 (1.f - 0.999f is 1.3e-5 away from float(1 - 0.999))
__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                   float* __restrict__ m, float* __restrict__ v, int64_t n,
                                                   const float* __restrict__ lr_p, const float* __restrict__ step_p,
                                                   double b1d, double b2d, double epsd, double wdd, int decoupled,
                                                   float gscale) {
  const float lr = *lr_p;
  const double step = (double)*step_p;
  const double bc1 = 1.0 - pow(b1d, step), bc2 = 1.0 - pow(b2d, step);
  const float step_size = (float)((double)lr / bc1), rbc2 = (float)(1.0 / sqrt(bc2));
  const float b1 = (float)b1d, b2 = (float)b2d, omb1 = (float)(1.0 - b1d), omb2 = (float)(1.0 - b2d);
  const float eps = (float)epsd, wd = (float)wdd, decay = (float)(1.0 - (double)lr * wdd);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float pi = p[i], gi = g[i] * gscale;
    if (wdd != 0.0) {
      if (decoupled) pi *= decay; else gi = fmaf(wd, pi, gi);
    }
    const float mi = fmaf(b1, m[i], omb1 * gi);
    const float vi = fmaf(b2, v[i], omb2 * gi * gi);
    m[i] = mi;
    v[i] = vi;
    p[i] = pi - step_size * mi / (sqrtf(vi) * rbc2 + eps);
  }
}

// ================================================================================================
// SGD
// ================================================================================================
// torch.optim.SGD's arithmetic: momentum and weight decay are cast to fp32 as torch does with python floats, (1 - dampening)
// is formed in double first.  The first step (buf = d, no dampening) is read from the device step counter, so a
// captured launch replays correctly after the eager warm-up step: step <= 1 means "no buffer yet".
__global__ void __launch_bounds__(256) sgd_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                  float* __restrict__ buf, int64_t n, const float* __restrict__ lr_p,
                                                  const float* __restrict__ step_p, double momd, double dampd,
                                                  double wdd, int nesterov, float gscale) {
  const float lr = *lr_p;
  const bool first = *step_p <= 1.f;
  const float mom = (float)momd, omd = (float)(1.0 - dampd), wd = (float)wdd;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float pi = p[i];
    float d = g[i] * gscale;
    if (wdd != 0.0) d = fmaf(wd, pi, d);
    if (momd != 0.0) {
      const float b = first ? d : fmaf(omd, d, mom * buf[i]);
      buf[i] = b;
      d = nesterov ? fmaf(mom, b, d) : b;
    }
    p[i] = fmaf(-lr, d, pi);
  }
}

__global__ void advance_seed_kernel(uint64_t* s) { *s += 1; }

}  // namespace seist

using namespace seist;

extern "C" {

int seist_bce_fwd(const float* preds, const float* targets, const float* weight, int64_t N, int32_t C, int64_t L,
                  float eps, double* loss_sum, float* loss_out, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t total = N * C * L;
  if (total <= 0) return -1;
  cudaMemsetAsync(loss_sum, 0, sizeof(double), s);
  bce_fwd_kernel<<<ew_grid(total), 256, 0, s>>>(preds, targets, weight, total, C, L, eps, loss_sum);
  note_launch();
  mean_finalize_kernel<<<1, 1, 0, s>>>(loss_sum, 1.0 / (double)total, loss_out);
  note_launch();
  return check_launch("bce_fwd");
}

int seist_bce_bwd(const float* preds, const float* targets, const float* weight, const float* gout, int64_t N,
                  int32_t C, int64_t L, float eps, float* dpreds, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t total = N * C * L;
  if (total <= 0) return -1;
  bce_bwd_kernel<<<ew_grid(total), 256, 0, s>>>(preds, targets, weight, gout, total, C, L, eps,
                                                (float)(1.0 / (double)total), dpreds);
  note_launch();
  return check_launch("bce_bwd");
}

int seist_ce_fwd(const float* preds, const float* targets, const float* weight, int64_t rows, int32_t C, float eps,
                 double* loss_sum, float* loss_out, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (rows <= 0 || C <= 0) return -1;
  cudaMemsetAsync(loss_sum, 0, sizeof(double), s);
  ce_fwd_kernel<<<ew_grid(rows * C), 256, 0, s>>>(preds, targets, weight, rows * C, C, eps, loss_sum);
  note_launch();
  mean_finalize_kernel<<<1, 1, 0, s>>>(loss_sum, 1.0 / (double)rows, loss_out);
  note_launch();
  return check_launch("ce_fwd");
}

int seist_ce_bwd(const float* preds, const float* targets, const float* weight, const float* gout, int64_t rows, int32_t C,
                 float eps, float* dpreds, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (rows <= 0 || C <= 0) return -1;
  ce_bwd_kernel<<<ew_grid(rows * C), 256, 0, s>>>(preds, targets, weight, gout, rows * C, C, eps, (float)(1.0 / (double)rows), dpreds);
  note_launch();
  return check_launch("ce_bwd");
}

int seist_huber_fwd(const float* preds, const float* targets, int64_t numel, float delta, double* loss_sum,
                    float* loss_out, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (numel <= 0) return -1;
  cudaMemsetAsync(loss_sum, 0, sizeof(double), s);
  huber_fwd_kernel<<<ew_grid(numel), 256, 0, s>>>(preds, targets, numel, delta, loss_sum);
  note_launch();
  mean_finalize_kernel<<<1, 1, 0, s>>>(loss_sum, 1.0 / (double)numel, loss_out);
  note_launch();
  return check_launch("huber_fwd");
}

int seist_huber_bwd(const float* preds, const float* targets, const float* gout, int64_t numel, float delta,
                    float* dpreds, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (numel <= 0) return -1;
  huber_bwd_kernel<<<ew_grid(numel), 256, 0, s>>>(preds, targets, gout, numel, delta, (float)(1.0 / (double)numel),
                                                  dpreds);
  note_launch();
  return check_launch("huber_bwd");
}

int seist_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t numel,
                    const float* lr, const float* step, double beta1, double beta2, double eps, double weight_decay,
                    int32_t decoupled, float grad_scale, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (numel <= 0) return -1;
  adam_kernel<<<ew_grid(numel), 256, 0, s>>>(params, grads, exp_avg, exp_avg_sq, numel, lr, step, beta1, beta2, eps,
                                             weight_decay, decoupled, grad_scale);
  note_launch();
  return check_launch("adam_step");
}

int seist_sgd_step(float* params, const float* grads, float* momentum_buf, int64_t numel, const float* lr,
                   const float* step, double momentum, double dampening, double weight_decay, int32_t nesterov,
                   float grad_scale, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (numel <= 0) return -1;
  if (momentum != 0.0 && momentum_buf == nullptr) { set_error("sgd_step: momentum needs a momentum buffer"); return -2; }
  if (nesterov && (momentum <= 0.0 || dampening != 0.0)) {
    set_error("sgd_step: nesterov needs a positive momentum and zero dampening");
    return -2;
  }
  sgd_kernel<<<ew_grid(numel), 256, 0, s>>>(params, grads, momentum_buf, numel, lr, step, momentum, dampening,
                                            weight_decay, nesterov, grad_scale);
  note_launch();
  return check_launch("sgd_step");
}

int seist_advance_seed(uint64_t* seed, void* stream) {
  advance_seed_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(seed);
  note_launch();
  return check_launch("advance_seed");
}

}  // extern "C"
