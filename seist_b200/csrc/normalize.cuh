// `DataPreprocessor._normalize` (reference training/preprocess.py:224-242) of one trace by one CTA of PR_NT threads, shared
// by the in-place batch normalisation (preproc.cu) and the window cut of continuous records (stream.cu), so that both
// produce the same bits.
#pragma once
#include "common.cuh"

namespace seist {

constexpr int PR_NT = 256;

static __device__ double pr_block_sum(double v, double* red_s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red_s[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < PR_NT / 32; ++w) s += red_s[w];
  return s;
}
static __device__ float pr_block_max(float v, float* red_s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red_s[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = red_s[0];
  for (int w = 1; w < PR_NT / 32; ++w) s = fmaxf(s, red_s[w]);
  return s;
}

// dst[i] = normalised src[i], i < L (src == dst allowed).  mode 0: mean removal only, 1: / std (population), 2: / max
// (signed maximum of the centred trace); zero scale -> 1.  Every thread of the CTA must call it.
static __device__ void pr_normalize_row(const float* src, float* dst, int L, int mode) {
  __shared__ double red_d[PR_NT / 32];
  __shared__ float red_f[PR_NT / 32];
  double s = 0.0;
  for (int i = threadIdx.x; i < L; i += PR_NT) s += (double)src[i];
  const float mean = (float)(pr_block_sum(s, red_d) / (double)L);
  float scale = 1.f;
  if (mode == 1) {
    double q = 0.0;
    for (int i = threadIdx.x; i < L; i += PR_NT) { const double d = (double)(src[i] - mean); q += d * d; }
    scale = (float)sqrt(pr_block_sum(q, red_d) / (double)L);
  } else if (mode == 2) {
    float m = -INFINITY;
    for (int i = threadIdx.x; i < L; i += PR_NT) m = fmaxf(m, src[i] - mean);
    scale = pr_block_max(m, red_f);
  }
  if (scale == 0.f) scale = 1.f;
  for (int i = threadIdx.x; i < L; i += PR_NT) dst[i] = (src[i] - mean) / scale;
}

}  // namespace seist
