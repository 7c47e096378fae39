// Input side on the device (SURVEY 8f-3): what the reference's DataLoader workers do per waveform in numpy
// (training/preprocess.py): `_normalize` (:224-242) and the dpk soft labels `_generate_soft_label` (:544-683) with
// `_pad_phases` (:16-35), all four window shapes.  One CTA per trace.  Floating point: double accumulation / double
// window evaluation, results within 2e-6 of the numpy oracle (oracle/preprocess_ref.py, bit-exactly pinned to the
// reference's own sources; the sigmoid window: tests/augment_ref.py).
#include "common.cuh"

namespace seist {

constexpr int PR_NT = 256;
constexpr int PR_MAXK = 8;
constexpr long long PR_ABSENT = -1000000;     // phase indices below this are "no phase" padding of the (N, K) index tensors

__device__ double pr_block_sum(double v, double* red_s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red_s[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < PR_NT / 32; ++w) s += red_s[w];
  return s;
}
__device__ float pr_block_max(float v, float* red_s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red_s[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = red_s[0];
  for (int w = 1; w < PR_NT / 32; ++w) s = fmaxf(s, red_s[w]);
  return s;
}

// mode 0: mean removal only, 1: / std (population), 2: / max (signed maximum of the centred trace); zero scale -> 1
__global__ void __launch_bounds__(PR_NT) normalize_rows_kernel(float* __restrict__ x, int L, int mode) {
  __shared__ double red_d[PR_NT / 32];
  __shared__ float red_f[PR_NT / 32];
  float* row = x + (size_t)blockIdx.x * L;
  double s = 0.0;
  for (int i = threadIdx.x; i < L; i += PR_NT) s += (double)row[i];
  const float mean = (float)(pr_block_sum(s, red_d) / (double)L);
  float scale = 1.f;
  if (mode == 1) {
    double q = 0.0;
    for (int i = threadIdx.x; i < L; i += PR_NT) { const double d = (double)(row[i] - mean); q += d * d; }
    scale = (float)sqrt(pr_block_sum(q, red_d) / (double)L);
  } else if (mode == 2) {
    float m = -INFINITY;
    for (int i = threadIdx.x; i < L; i += PR_NT) m = fmaxf(m, row[i] - mean);
    scale = pr_block_max(m, red_f);
  }
  if (scale == 0.f) scale = 1.f;
  for (int i = threadIdx.x; i < L; i += PR_NT) row[i] = (row[i] - mean) / scale;
}

__device__ __forceinline__ double pr_window(int d, int left, int right, int width, int shape) {
  if (d < -left || d > right) return 0.0;
  if (shape == 0) return exp(-((double)d * (double)d) / 200.0);                     // gaussian, sigma 10 samples
  if (shape == 1) return 1.0 - fabs(2.0 / (double)width * (double)d);               // triangle
  if (shape == 3) {                                                                 // sigmoid (:586-597)
    if (d == 0) return 1.0;
    // left shoulder: 1 / (1 + exp(-10 / left * a)), a = -int(left / 2) + (d + left); right: 10 / right * a, a from
    // -int(right / 2) at d = 1
    const double a = d < 0 ? (double)(d + left - left / 2) : (double)(d - 1 - right / 2);
    const double xv = d < 0 ? __dmul_rn(-10.0 / (double)left, a) : __dmul_rn(-10.0 / (double)right * -1.0, a);
    return 1.0 / __dadd_rn(1.0, exp(xv));
  }
  return 1.0;                                                                       // box
}
__device__ __forceinline__ double pr_soft(const long long* idx, int n, int j, int L, int left, int right, int width, int shape) {
  double s = 0.0;
  for (int i = 0; i < n; ++i) {
    const long long c = idx[i];
    if (c < 0 || c > L - 1) continue;
    s += pr_window(j - (int)c, left, right, width, shape);
  }
  return s;
}

// out (N, 3, L): det, ppk, spk
__global__ void __launch_bounds__(PR_NT) dpk_labels_kernel(const long long* __restrict__ ppks, const long long* __restrict__ spks, int K,
                                                           int L, int width, int shape, double coda_ratio, float* __restrict__ out) {
  __shared__ long long p_s[PR_MAXK], s_s[PR_MAXK], pp_s[2 * PR_MAXK], ss_s[2 * PR_MAXK];
  __shared__ int np_s, ns_s, npair_s;
  const int n = blockIdx.x;
  if (threadIdx.x == 0) {
    int np = 0, ns = 0;
    for (int i = 0; i < K; ++i) {
      if (ppks[(size_t)n * K + i] > PR_ABSENT) p_s[np++] = ppks[(size_t)n * K + i];
      if (spks[(size_t)n * K + i] > PR_ABSENT) s_s[ns++] = spks[(size_t)n * K + i];
    }
    for (int i = 1; i < np; ++i) { long long v = p_s[i]; int j = i - 1; while (j >= 0 && p_s[j] > v) { p_s[j + 1] = p_s[j]; --j; } p_s[j + 1] = v; }
    for (int i = 1; i < ns; ++i) { long long v = s_s[i]; int j = i - 1; while (j >= 0 && s_s[j] > v) { s_s[j + 1] = s_s[j]; --j; } s_s[j + 1] = v; }
    // _pad_phases (:16-35): the largest idx such that the first idx+1 P picks all precede the last idx+1 S picks
    int idx = 0;
    const int mn = np < ns ? np : ns;
    while (idx < mn) {
      bool all_lt = true;
      for (int a = 0; a <= idx; ++a) all_lt = all_lt && (p_s[a] < s_s[ns - idx - 1 + a]);
      if (!all_lt) break;
      ++idx;
    }
    int m = 0;
    for (int a = 0; a < ns - idx; ++a) pp_s[m++] = -(long long)(width < 0 ? -width : width);
    for (int a = 0; a < np; ++a) pp_s[m++] = p_s[a];
    int m2 = 0;
    for (int a = 0; a < ns; ++a) ss_s[m2++] = s_s[a];
    for (int a = idx; a < np; ++a) ss_s[m2++] = (long long)L + (width < 0 ? -width : width);
    np_s = np; ns_s = ns; npair_s = m < m2 ? m : m2;
  }
  __syncthreads();
  const int left = width / 2, right = width - left;
  float* o = out + (size_t)n * 3 * L;
  for (int j = threadIdx.x; j < L; j += PR_NT) {
    double det = 0.0;
    for (int a = 0; a < npair_s; ++a) {
      const long long ppk = pp_s[a], spk = ss_s[a];
      const long long dte = (long long)((double)spk + coda_ratio * (double)(spk - ppk));   // python int(): truncation, in double
      const long long two[2] = {ppk, dte};
      double li = pr_soft(two, 2, j, L, left, right, width, shape);
      const long long c0 = ppk < 0 ? 0 : (ppk > L ? L : ppk), c1 = dte < 0 ? 0 : (dte > L ? L : dte);
      if (j >= c0 && j < c1) li = 1.0;
      det += li;
    }
    o[j] = (float)(det > 1.0 ? 1.0 : det);
    o[L + j] = (float)pr_soft(p_s, np_s, j, L, left, right, width, shape);
    o[2 * (size_t)L + j] = (float)pr_soft(s_s, ns_s, j, L, left, right, width, shape);
  }
}

}  // namespace seist

using namespace seist;

extern "C" {

int seist_normalize(float* x, int64_t rows, int32_t L, int32_t mode, void* stream) {
  if (!x || rows <= 0 || L <= 0 || mode < 0 || mode > 2) { set_error("normalize: bad arguments (mode 0 none, 1 std, 2 max)"); return -1; }
  normalize_rows_kernel<<<(unsigned)rows, PR_NT, 0, (cudaStream_t)stream>>>(x, L, mode);
  note_launch();
  return check_launch("normalize");
}

int seist_dpk_labels(const int64_t* ppks, const int64_t* spks, int64_t N, int32_t K, int32_t L, int32_t width, int32_t shape,
                     double coda_ratio, float* out, void* stream) {
  if (!ppks || !spks || !out || N <= 0 || K < 1 || K > PR_MAXK || L <= 0 || width < 1 || shape < 0 || shape > 3 ||
      (shape == 3 && width < 2)) {
    set_error("dpk_labels: bad arguments (1 <= K <= 8, shape 0 gaussian / 1 triangle / 2 box / 3 sigmoid with width >= 2)");
    return -1;
  }
  dpk_labels_kernel<<<(unsigned)N, PR_NT, 0, (cudaStream_t)stream>>>((const long long*)ppks, (const long long*)spks, K, L, width, shape,
                                                                    coda_ratio, out);
  note_launch();
  return check_launch("dpk_labels");
}

}  // extern "C"
