// Continuous records on the device: sliding-window inference input, overlap stacking of the window outputs and
// whole-record peak picking / event runs (DESIGN §4.15).  The reference has no continuous-data path (demo_predict.py:75
// keeps the first 8192 samples); per window it is `_normalize` (training/preprocess.py:224-242) -> model -> per trace
// `_detect_peaks` (training/postprocess.py:15-111, topk = None) and obspy `trigger_onset(p, thr, thr)` (:114-158).
//
// Windows of a station of T samples: starts k * P for k = 0 .. Kr - 1, Kr = (T - W) / P + 1, plus one start at T - W
// when the last of those ends before T; K windows per station, window id s * K + k.
#include <algorithm>

#include "normalize.cuh"

namespace seist {

constexpr int ST_NT = 256;
constexpr int ST_CH = ST_NT * 16;      // elements per block of the count / fill passes
constexpr int ST_SCAN_NT = 1024;
constexpr int CL_SEG = 1024;           // candidates whose cluster starts a CTA of the cluster pass looks at
constexpr int CL_SMALL = 32;           // clusters up to this size are resolved by one thread
constexpr int CL_SMEM = 4096;          // largest cluster staged in shared memory; larger ones stay in global memory
constexpr unsigned char CL_OPEN = 0, CL_KEEP = 1, CL_DROP = 2;

struct Windows {
  int T, W, P, Kr, K;
  __host__ __device__ Windows(int T_, int W_, int P_) : T(T_), W(W_), P(P_) {
    Kr = (T - W) / P + 1;
    K = Kr + ((long long)(Kr - 1) * P + W < T ? 1 : 0);
  }
  __host__ __device__ int start(int k) const { return k < Kr ? k * P : T - W; }
  // covering windows of sample t: the regular ones [lo, hi] (empty when lo > hi), then the tail window K - 1 if
  // t >= T - W and it exists
  __device__ void cover(int t, int& lo, int& hi, bool& tail) const {
    lo = t < W ? 0 : (t - W) / P + 1;
    hi = min(Kr - 1, t / P);
    tail = K > Kr && t >= T - W;
  }
};

// ---- window batch -------------------------------------------------------------------------------------------------
// x (B, C, W): row (b, c) = normalised record[s, c, start(k):start(k)+W] for window w0 + b = s * K + k; zero past S * K.
__global__ void __launch_bounds__(PR_NT) window_batch_kernel(const float* __restrict__ rec, int S, int C, Windows win,
                                                             long long w0, int mode, float* __restrict__ x) {
  extern __shared__ float wb_row[];                 // [W]: the record slice, read from global memory once
  const int b = blockIdx.x / C, c = blockIdx.x % C;
  const long long w = w0 + b;
  float* dst = x + (size_t)blockIdx.x * win.W;
  if (w >= (long long)S * win.K) {
    for (int i = threadIdx.x; i < win.W; i += PR_NT) dst[i] = 0.f;
    return;
  }
  const int s = (int)(w / win.K), k = (int)(w % win.K);
  const float* src = rec + ((size_t)s * C + c) * win.T + win.start(k);
  for (int i = threadIdx.x; i < win.W; i += PR_NT) wb_row[i] = src[i];
  __syncthreads();
  pr_normalize_row(wb_row, dst, win.W, mode);
}

// ---- P-anchored event windows (DESIGN §4.17) ----------------------------------------------------------------------
// `_cut_window` with 0 <= p_position_ratio <= 1 (training/preprocess.py:172-203) then `_normalize` of every P pick of a
// CSR pick list.  x_d (B, C, W), d < n_dst: row (b, c) = normalised record[s, c, p - a + i], i < W, 0.0f where p - a + i
// falls outside [0, T); p = index[e0 + b], s the station whose offsets range holds event e0 + b.  Events >= M and picks
// outside [0, T) give zero rows.
constexpr int EW_MAX_DST = 4;
struct EventDst {
  float* x[EW_MAX_DST];
};

__global__ void __launch_bounds__(PR_NT) event_windows_kernel(const float* __restrict__ rec, int S, int C, int T,
                                                              const long long* __restrict__ index,
                                                              const long long* __restrict__ offsets, long long M, long long e0,
                                                              int W, int a, int mode, EventDst dst, int n_dst) {
  extern __shared__ float ew_row[];                 // [W]: the zero-filled record slice, normalised in place
  const int b = blockIdx.x / C, c = blockIdx.x % C;
  const long long e = e0 + b;
  const size_t row = (size_t)blockIdx.x * W;
  const long long p = e < M ? index[e] : -1;
  if (p < 0 || p >= T) {
#pragma unroll
    for (int d = 0; d < EW_MAX_DST; ++d)           // unrolled: a runtime index into dst would put it on the stack
      if (d < n_dst)
        for (int i = threadIdx.x; i < W; i += PR_NT) dst.x[d][row + i] = 0.f;
    return;
  }
  // the last station s with offsets[s] <= e (empty stations before it share its start); always in [0, S), so
  // malformed offsets pick a wrong station but never an out-of-range one
  int lo = 0, hi = S - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (offsets[mid] <= e) lo = mid; else hi = mid - 1;
  }
  const float* src = rec + ((size_t)lo * C + c) * T;
  const long long t0 = p - a;
  for (int i = threadIdx.x; i < W; i += PR_NT) {
    const long long t = t0 + i;
    ew_row[i] = t >= 0 && t < T ? src[t] : 0.f;
  }
  __syncthreads();
  pr_normalize_row(ew_row, ew_row, W, mode);
  // each thread stores the elements it normalised itself: no barrier needed
#pragma unroll
  for (int d = 0; d < EW_MAX_DST; ++d)
    if (d < n_dst)
      for (int i = threadIdx.x; i < W; i += PR_NT) dst.x[d][row + i] = ew_row[i];
}

// ---- stacking -----------------------------------------------------------------------------------------------------
// Gather: the thread of probs[s, c, t] adds (maxes) the batch's covering windows of t in ascending window order; the
// first covering window of t overall starts the accumulator (0.0f + v for the mean, fmaxf(-inf, v) for the max).
__global__ void __launch_bounds__(ST_NT) stack_batch_kernel(const float* __restrict__ y, int S, Windows win, long long w0,
                                                            int nb, int s0, int mode, float* __restrict__ probs) {
  const int s = s0 + blockIdx.y, c = blockIdx.z;
  const long long wb = (long long)s * win.K;
  const int ka = (int)max(w0 - wb, 0LL), kb = (int)min(w0 + nb - 1 - wb, (long long)win.K - 1);
  if (s >= S || ka > kb) return;
  const int t = win.start(ka) + blockIdx.x * ST_NT + threadIdx.x;
  if (t >= win.start(kb) + win.W) return;
  int lo, hi;
  bool tail;
  win.cover(t, lo, hi, tail);
  const int first = lo <= hi ? lo : win.K - 1;
  float* out = probs + ((size_t)s * 3 + c) * win.T + t;
  float acc = first >= ka ? (mode == 0 ? 0.f : -INFINITY) : *out;
  const float* yb = y + (size_t)c * win.W;
  for (int k = max(lo, ka); k <= min(hi, kb); ++k) {
    const float v = yb[(size_t)(wb + k - w0) * 3 * win.W + (t - k * win.P)];
    acc = mode == 0 ? acc + v : fmaxf(acc, v);
  }
  if (tail && win.K - 1 >= ka && win.K - 1 <= kb) {
    const float v = yb[(size_t)(wb + win.K - 1 - w0) * 3 * win.W + (t - (win.T - win.W))];
    acc = mode == 0 ? acc + v : fmaxf(acc, v);
  }
  *out = acc;
}

// mean: one IEEE division by the number of covering windows
__global__ void __launch_bounds__(ST_NT) stack_finish_kernel(float* __restrict__ probs, Windows win, long long n) {
  for (long long i = blockIdx.x * (long long)ST_NT + threadIdx.x; i < n; i += (long long)gridDim.x * ST_NT) {
    int lo, hi;
    bool tail;
    win.cover((int)(i % win.T), lo, hi, tail);
    const int cnt = max(hi - lo + 1, 0) + (tail ? 1 : 0);
    probs[i] = __fdiv_rn(probs[i], (float)cnt);
  }
}

// ---- order-preserving compaction: per-block counts, a per-row scan of the counts, a fill pass --------------------
// exclusive rank of this thread's flag among the CTA's flags of one step, and the step's total
__device__ __forceinline__ int st_block_rank(bool f, int* warp_s, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, f);
  __syncthreads();
  if (lane == 0) warp_s[warp] = __popc(m);
  __syncthreads();
  int base = 0;
  total = 0;
  for (int w = 0; w < ST_NT / 32; ++w) {
    if (w < warp) base += warp_s[w];
    total += warp_s[w];
  }
  return base + __popc(m & ((1u << lane) - 1u));
}

__device__ __forceinline__ int st_block_count(int v, int* warp_s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) warp_s[threadIdx.x >> 5] = v;
  __syncthreads();
  int s = 0;
  for (int w = 0; w < ST_NT / 32; ++w) s += warp_s[w];
  return s;
}

// blk (rows, nblk): counts -> exclusive offsets in place; total[row]; total64[row] too when given
__global__ void __launch_bounds__(ST_SCAN_NT) scan_rows_kernel(int* __restrict__ blk, int nblk, int* __restrict__ total,
                                                               long long* __restrict__ total64) {
  __shared__ int warp_s[ST_SCAN_NT / 32];
  __shared__ int carry_s;
  int* row = blk + (size_t)blockIdx.x * nblk;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (int base = 0; base < nblk; base += ST_SCAN_NT) {
    const int i = base + threadIdx.x;
    const int v = i < nblk ? row[i] : 0;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += u;
    }
    if (lane == 31) warp_s[warp] = inc;
    __syncthreads();
    int wbase = 0, tot = 0;
    for (int w = 0; w < ST_SCAN_NT / 32; ++w) {
      if (w < warp) wbase += warp_s[w];
      tot += warp_s[w];
    }
    const int carry = carry_s;
    if (i < nblk) row[i] = carry + wbase + inc - v;
    __syncthreads();
    if (threadIdx.x == 0) carry_s = carry + tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    total[blockIdx.x] = carry_s;
    if (total64) total64[blockIdx.x] = carry_s;
  }
}

// ---- peaks --------------------------------------------------------------------------------------------------------
// rising-edge peak candidate (postprocess.py:67-68,82-88): x[i] - x[i-1] > 0, x[i+1] - x[i] <= 0, x[i] >= mph; the callers
// test i in [lo, hi] only (1 .. T - 2 of a whole row; the newly decided samples of a streamed row)
__device__ __forceinline__ bool pk_cand(const float* x, int i, float mph) {
  const float v = x[i];
  return v - x[i - 1] > 0.f && x[i + 1] - v <= 0.f && v >= mph;
}

// blocks of ST_CH samples from lo; blk (rows, nblk)
__global__ void __launch_bounds__(ST_NT) cand_count_kernel(const float* __restrict__ prob, long long n_stride, int lo, int hi, float mph,
                                                           int* __restrict__ blk, int nblk) {
  __shared__ int warp_s[ST_NT / 32];
  const float* x = prob + blockIdx.y * n_stride;
  const int a = lo + blockIdx.x * ST_CH;
  int n = 0;
  for (int i = a + threadIdx.x; i < min(a + ST_CH, hi + 1); i += ST_NT) n += pk_cand(x, i, mph);
  n = st_block_count(n, warp_s);
  if (threadIdx.x == 0) blk[(size_t)blockIdx.y * nblk + blockIdx.x] = n;
}

// candidate i goes to cidx[row, off0[row] + rank] (off0 may be null: 0) as i + ishift
__global__ void __launch_bounds__(ST_NT) cand_fill_kernel(const float* __restrict__ prob, long long n_stride, int lo, int hi, float mph,
                                                          const int* __restrict__ blk, int nblk, const int* __restrict__ off0, int ishift,
                                                          int capc, int* __restrict__ cidx, float* __restrict__ cval) {
  __shared__ int warp_s[ST_NT / 32];
  const float* x = prob + blockIdx.y * n_stride;
  const int a = lo + blockIdx.x * ST_CH;
  int base = blk[(size_t)blockIdx.y * nblk + blockIdx.x] + (off0 ? off0[blockIdx.y] : 0);
  int* ci = cidx + (size_t)blockIdx.y * capc;
  float* cv = cval + (size_t)blockIdx.y * capc;
  for (int i0 = a; i0 < min(a + ST_CH, hi + 1); i0 += ST_NT) {
    const int i = i0 + threadIdx.x;
    const bool f = i <= hi && pk_cand(x, i, mph);
    int tot;
    const int r = st_block_rank(f, warp_s, tot);
    if (f) { ci[base + r] = i + ishift; cv[base + r] = x[i]; }
    base += tot;
  }
}

// ranked before: higher value, equal values: larger sample index (oracle/postprocess_ref.py tie rule)
__device__ __forceinline__ bool pk_above(float vq, int iq, float vk, int ik) { return vq > vk || (vq == vk && iq > ik); }

// Decide candidate k of a cluster if its neighbours within mpd allow it: dropped once a higher-ranked one is kept, kept
// once every higher-ranked one is dropped.
__device__ __forceinline__ unsigned char pk_decide(const int* ci, const float* cv, volatile unsigned char* st, int m, int k, int mpd) {
  const int ik = ci[k];
  const float vk = cv[k];
  bool open = false;
  for (int q = k - 1; q >= 0 && ik - ci[q] <= mpd; --q) {
    if (!pk_above(cv[q], ci[q], vk, ik)) continue;
    const unsigned char sq = st[q];
    if (sq == CL_KEEP) return CL_DROP;
    open = open || sq == CL_OPEN;
  }
  for (int q = k + 1; q < m && ci[q] - ik <= mpd; ++q) {
    if (!pk_above(cv[q], ci[q], vk, ik)) continue;
    const unsigned char sq = st[q];
    if (sq == CL_KEEP) return CL_DROP;
    open = open || sq == CL_OPEN;
  }
  return open ? CL_OPEN : CL_KEEP;
}

// Greedy suppression of one cluster of m candidates by the whole CTA, as the fixed point of pk_decide.  Decisions are
// final and only follow from decided neighbours, so a thread may act on neighbours' states of any age: each thread
// sweeps its contiguous share both ways until it stalls, then the CTA synchronises.  Every round decides at least the
// highest-ranked open candidate.  ci / cv / st are in shared or global memory.
__device__ void pk_cluster_cta(const int* ci, const float* cv, volatile unsigned char* st, int m, int mpd) {
  const int lo = (int)((long long)m * threadIdx.x / ST_NT), hi = (int)((long long)m * (threadIdx.x + 1) / ST_NT);
  for (;;) {
    bool changed = true, open = false;
    while (changed) {
      changed = false;
      for (int k = lo; k < hi; ++k)
        if (st[k] == CL_OPEN) {
          const unsigned char d = pk_decide(ci, cv, st, m, k, mpd);
          if (d != CL_OPEN) { st[k] = d; changed = true; }
        }
      for (int k = hi - 1; k >= lo; --k)
        if (st[k] == CL_OPEN) {
          const unsigned char d = pk_decide(ci, cv, st, m, k, mpd);
          if (d != CL_OPEN) { st[k] = d; changed = true; }
        }
    }
    for (int k = lo; k < hi; ++k) open = open || st[k] == CL_OPEN;
    if (!__syncthreads_or(open)) break;
  }
}

// Clusters: maximal runs of candidates whose consecutive gaps are <= mpd; a candidate suppresses or is suppressed only
// inside its cluster.  CTA (seg, row) resolves the clusters that start among candidates [seg * CL_SEG, +CL_SEG): small
// ones one per thread (greedy in height order), the others together.
__global__ void __launch_bounds__(ST_NT) cluster_kernel(const int* __restrict__ ncand, int capc, const int* cidx, const float* cval,
                                                        unsigned char* state, int mpd) {
  __shared__ int ci_s[CL_SMEM];
  __shared__ float cv_s[CL_SMEM];
  __shared__ unsigned char st_s[CL_SMEM];
  __shared__ int big_s[CL_SEG];
  __shared__ int nbig_s, end_s;
  const int n = ncand[blockIdx.y];
  const int a = blockIdx.x * CL_SEG;
  if (a >= n) return;
  const int b = min(a + CL_SEG, n);
  const int* ci = cidx + (size_t)blockIdx.y * capc;
  const float* cv = cval + (size_t)blockIdx.y * capc;
  unsigned char* st = state + (size_t)blockIdx.y * capc;
  if (threadIdx.x == 0) nbig_s = 0;
  __syncthreads();
  for (int j = a + threadIdx.x; j < b; j += ST_NT) {
    if (j > 0 && ci[j] - ci[j - 1] <= mpd) continue;          // not the first of its cluster
    int e = j;
    while (e + 1 < n && ci[e + 1] - ci[e] <= mpd && e - j < CL_SMALL) ++e;
    if (e - j == CL_SMALL) { big_s[atomicAdd(&nbig_s, 1)] = j; continue; }
    for (int k = j; k <= e; ++k) st[k] = CL_OPEN;
    for (;;) {                                                // greedy: keep the best open one, drop its open neighbours
      int best = -1;
      for (int k = j; k <= e; ++k)
        if (st[k] == CL_OPEN && (best < 0 || pk_above(cv[k], ci[k], cv[best], ci[best]))) best = k;
      if (best < 0) break;
      st[best] = CL_KEEP;
      for (int k = j; k <= e; ++k)
        if (st[k] == CL_OPEN && abs(ci[k] - ci[best]) <= mpd) st[k] = CL_DROP;
    }
  }
  __syncthreads();
  const int nbig = nbig_s;
  for (int q = 0; q < nbig; ++q) {
    const int j = big_s[q];
    if (threadIdx.x == 0) end_s = n - 1;
    __syncthreads();
    for (int base = j; base < n - 1; base += ST_NT) {         // the cluster ends before the first gap > mpd
      const int k = base + threadIdx.x;
      if (k < n - 1 && ci[k + 1] - ci[k] > mpd) atomicMin(&end_s, k);
      if (__syncthreads_or(end_s < n - 1)) break;
    }
    const int m = end_s - j + 1;
    if (m <= CL_SMEM) {
      for (int k = threadIdx.x; k < m; k += ST_NT) { ci_s[k] = ci[j + k]; cv_s[k] = cv[j + k]; st_s[k] = CL_OPEN; }
      __syncthreads();
      pk_cluster_cta(ci_s, cv_s, st_s, m, mpd);
      for (int k = threadIdx.x; k < m; k += ST_NT) st[j + k] = st_s[k];
    } else {
      for (int k = threadIdx.x; k < m; k += ST_NT) st[j + k] = CL_OPEN;
      __syncthreads();
      pk_cluster_cta(ci + j, cv + j, st + j, m, mpd);
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(ST_NT) keep_count_kernel(const int* __restrict__ ncand, int capc, const unsigned char* __restrict__ state,
                                                           int* __restrict__ blk, int nblk) {
  __shared__ int warp_s[ST_NT / 32];
  const int n = ncand[blockIdx.y];
  const unsigned char* st = state + (size_t)blockIdx.y * capc;
  const int a = blockIdx.x * ST_CH;
  int c = 0;
  for (int j = a + threadIdx.x; j < min(a + ST_CH, n); j += ST_NT) c += st[j] == CL_KEEP;
  c = st_block_count(c, warp_s);
  if (threadIdx.x == 0) blk[(size_t)blockIdx.y * nblk + blockIdx.x] = c;
}

__global__ void __launch_bounds__(ST_NT) keep_fill_kernel(const int* __restrict__ ncand, int capc, const int* __restrict__ cidx,
                                                          const float* __restrict__ cval, const unsigned char* __restrict__ state,
                                                          const int* __restrict__ blk, int nblk, const long long* __restrict__ offsets,
                                                          long long ishift, long long* __restrict__ index, float* __restrict__ value) {
  __shared__ int warp_s[ST_NT / 32];
  const int n = ncand[blockIdx.y];
  const int a = blockIdx.x * ST_CH;
  if (a >= n) return;
  const size_t r0 = (size_t)blockIdx.y * capc;
  long long base = offsets[blockIdx.y] + blk[(size_t)blockIdx.y * nblk + blockIdx.x];
  for (int j0 = a; j0 < min(a + ST_CH, n); j0 += ST_NT) {
    const int j = j0 + threadIdx.x;
    const bool f = j < n && state[r0 + j] == CL_KEEP;
    int tot;
    const int r = st_block_rank(f, warp_s, tot);
    if (f) { index[base + r] = cidx[r0 + j] + ishift; value[base + r] = cval[r0 + j]; }
    base += tot;
  }
}

// ---- runs of p > thr ----------------------------------------------------------------------------------------------
__device__ __forceinline__ bool rn_on(const float* x, int i, float thr) { return x[i] > thr && (i == 0 || !(x[i - 1] > thr)); }
__device__ __forceinline__ bool rn_off(const float* x, int i, int T, float thr) { return x[i] > thr && (i == T - 1 || !(x[i + 1] > thr)); }

__global__ void __launch_bounds__(ST_NT) run_count_kernel(const float* __restrict__ prob, long long n_stride, int T, float thr,
                                                          int* __restrict__ blk, int nblk) {
  __shared__ int warp_s[ST_NT / 32];
  const float* x = prob + blockIdx.y * n_stride;
  const int a = blockIdx.x * ST_CH;
  int n = 0;
  for (int i = a + threadIdx.x; i < min(a + ST_CH, T); i += ST_NT) n += rn_on(x, i, thr);
  n = st_block_count(n, warp_s);
  if (threadIdx.x == 0) blk[(size_t)blockIdx.y * nblk + blockIdx.x] = n;
}

// blk holds the exclusive run-start offsets per block; the offs before a block are as many, less one when a run crosses
// into the block
__global__ void __launch_bounds__(ST_NT) run_fill_kernel(const float* __restrict__ prob, long long n_stride, int T, float thr,
                                                         const int* __restrict__ blk, int nblk, const long long* __restrict__ offsets,
                                                         long long* __restrict__ pairs) {
  __shared__ int warp_s[ST_NT / 32];
  const float* x = prob + blockIdx.y * n_stride;
  const int a = blockIdx.x * ST_CH;
  const long long b0 = offsets[blockIdx.y] + blk[(size_t)blockIdx.y * nblk + blockIdx.x];
  long long on_base = b0, off_base = b0 - (a > 0 && x[a - 1] > thr && x[a] > thr ? 1 : 0);
  for (int i0 = a; i0 < min(a + ST_CH, T); i0 += ST_NT) {
    const int i = i0 + threadIdx.x;
    const bool fon = i < T && rn_on(x, i, thr), foff = i < T && rn_off(x, i, T, thr);
    int ton, toff;
    const int ron = st_block_rank(fon, warp_s, ton);
    const int roff = st_block_rank(foff, warp_s, toff);
    if (fon) pairs[(on_base + ron) * 2] = i;
    if (foff) pairs[(off_base + roff) * 2 + 1] = i;
    on_base += ton;
    off_base += toff;
  }
}

// ---- streamed records (DESIGN §4.16) -------------------------------------------------------------------------------
// One call of a stream is a SeistStreamStep (include/seist_b200.h); every sample index is a global int64 count.
__device__ __forceinline__ int ss_nw(const SeistStreamStep& p) { return p.nk + (p.tail >= 0 ? 1 : 0); }
__device__ __forceinline__ long long ss_start(const SeistStreamStep& p, int q) { return q < p.nk ? (p.k0 + q) * (long long)p.P : p.tail; }

// raw sample g of (s, c): the chunk from r0 on, the kept tail [r0 - min(W, r0), r0) before
__device__ __forceinline__ float ss_raw(const SeistStreamStep& p, const float* tail, const float* chunk, int s, int c, long long g) {
  if (g >= p.r0) return chunk[((size_t)s * p.C + c) * (size_t)(p.r1 - p.r0) + (size_t)(g - p.r0)];
  return tail[((size_t)s * p.C + c) * p.W + (size_t)(g - (p.r0 - min((long long)p.W, (long long)p.r0)))];
}

// x (B, C, W): row (b, c) = normalised window j0 + b of the call; zero past the call's last window
__global__ void __launch_bounds__(PR_NT) stream_window_kernel(SeistStreamStep p, const float* __restrict__ tail,
                                                              const float* __restrict__ chunk, long long j0, float* __restrict__ x) {
  extern __shared__ float sw_row[];                 // [W]
  const int b = blockIdx.x / p.C, c = blockIdx.x % p.C;
  const long long j = j0 + b;
  const int nw = ss_nw(p);
  float* dst = x + (size_t)blockIdx.x * p.W;
  if (j >= (long long)p.S * nw) {
    for (int i = threadIdx.x; i < p.W; i += PR_NT) dst[i] = 0.f;
    return;
  }
  const int s = (int)(j / nw);
  const long long a = ss_start(p, (int)(j % nw));
  for (int i = threadIdx.x; i < p.W; i += PR_NT) sw_row[i] = ss_raw(p, tail, chunk, s, c, a + i);
  __syncthreads();
  pr_normalize_row(sw_row, dst, p.W, p.norm_mode);
}

// tail_out (S, C, W): the last min(W, r1) raw samples after the call
__global__ void __launch_bounds__(ST_NT) stream_keep_kernel(SeistStreamStep p, const float* __restrict__ tail,
                                                            const float* __restrict__ chunk, float* __restrict__ tail_out) {
  const int s = blockIdx.y / p.C, c = blockIdx.y % p.C;
  const long long keep = min((long long)p.W, (long long)p.r1);
  const int i = blockIdx.x * ST_NT + threadIdx.x;
  if (i < keep) tail_out[(size_t)blockIdx.y * p.W + i] = ss_raw(p, tail, chunk, s, c, p.r1 - keep + i);
}

// stack_batch_kernel for the call's windows j0 .. j0 + nb - 1 into acc ([f0, r1)).  A sample that is not new continues
// from acc when an earlier batch of the call covered it (the station's part of the batch starts after the call's first
// window: the window before it covers t), else from carry ([f0, r0), earlier calls)
__global__ void __launch_bounds__(ST_NT) stream_stack_kernel(SeistStreamStep p, const float* __restrict__ y, long long j0, int nb, int s0,
                                                             const float* __restrict__ carry, float* __restrict__ acc) {
  const int s = s0 + blockIdx.y, c = blockIdx.z;
  const int nw = ss_nw(p);
  const long long wb = (long long)s * nw;
  const int qa = (int)max(j0 - wb, 0LL), qb = (int)min(j0 + nb - 1 - wb, (long long)nw - 1);
  if (s >= p.S || qa > qb) return;
  const long long t = ss_start(p, qa) + blockIdx.x * (long long)ST_NT + threadIdx.x;
  if (t >= ss_start(p, qb) + p.W) return;
  const long long lo = t < p.W ? 0 : (t - p.W) / p.P + 1, hi = min(t / p.P, (long long)p.k0 + p.nk - 1);
  const bool reg = lo <= hi;                                   // else the tail window is t's only one
  const bool tl = p.tail >= 0 && qb == nw - 1 && t >= p.tail;
  const long long kqa = p.k0 + qa;
  const bool first = reg ? (qa < p.nk && lo >= kqa) : tl;
  float* out = acc + ((size_t)s * 3 + c) * (size_t)(p.r1 - p.f0) + (size_t)(t - p.f0);
  float a = first ? (p.stack_mode == 0 ? 0.f : -INFINITY)
                  : (qa > 0 ? *out : carry[((size_t)s * 3 + c) * p.W + (size_t)(t - p.f0)]);   // window k0 + qa - 1 covers t
  const float* yb = y + (size_t)c * p.W;
  const long long kb = min(hi, (long long)p.k0 + min(qb, p.nk - 1));
  for (long long k = max(lo, kqa); k <= kb; ++k) {
    const float v = yb[(size_t)(wb + (k - p.k0) - j0) * 3 * p.W + (size_t)(t - k * p.P)];
    a = p.stack_mode == 0 ? a + v : fmaxf(a, v);
  }
  if (tl) {
    const float v = yb[(size_t)(wb + p.nk - j0) * 3 * p.W + (size_t)(t - p.tail)];
    a = p.stack_mode == 0 ? a + v : fmaxf(a, v);
  }
  *out = a;
}

// probs = final [f0, f1) (the mean divided once by its number of covering windows), carry_out = partial sums of [f1, r1)
__global__ void __launch_bounds__(ST_NT) stream_emit_kernel(SeistStreamStep p, const float* __restrict__ carry, const float* __restrict__ acc,
                                                            float* __restrict__ probs, float* __restrict__ carry_out) {
  const long long L = p.r1 - p.f0, n = (long long)p.S * 3 * L;
  const long long run_lo = p.k0 * p.P, run_hi = (p.k0 + p.nk - 1) * p.P + p.W;
  for (long long i = blockIdx.x * (long long)ST_NT + threadIdx.x; i < n; i += (long long)gridDim.x * ST_NT) {
    const long long row = i / L, t = p.f0 + i % L;
    const bool touched = (p.nk > 0 && t >= run_lo && t < run_hi) || (p.tail >= 0 && t >= p.tail);
    float v = touched ? acc[i] : (t < p.r0 ? carry[row * p.W + (t - p.f0)] : 0.f);   // t >= r0 untouched: no window yet
    if (t < p.f1) {
      if (p.stack_mode == 0) {
        const long long lo = t < p.W ? 0 : (t - p.W) / p.P + 1, hi = p.kr >= 0 ? min(t / p.P, (long long)p.kr - 1) : t / p.P;
        const int cnt = (int)max(hi - lo + 1, 0LL) + (p.tail >= 0 && t >= p.tail ? 1 : 0);
        v = __fdiv_rn(v, (float)cnt);
      }
      probs[row * (p.f1 - p.f0) + (t - p.f0)] = v;
    } else {
      carry_out[row * p.W + (t - p.f1)] = v;
    }
  }
}

// runs of a streamed row: position p closes a run at p - 1 (sr_off) or opens one at p (sr_on); x[lo - 1] is the last
// sample of the previous stretch
__device__ __forceinline__ bool sr_off(const float* x, int p, float thr) { return x[p - 1] > thr && !(x[p] > thr); }
__device__ __forceinline__ bool sr_on(const float* x, int p, float thr) { return x[p] > thr && !(x[p - 1] > thr); }

// ---- ragged streams: stations that advance at different rates (DESIGN §4.19) ----------------------------------------
// One SeistRaggedStep per call; the per-station counts are device arrays, the call's data packed by the prefix arrays.

// the last row r in [0, n) with off[r] <= j: the row whose packed range holds j (empty rows before it share its start);
// always in [0, n), so malformed offsets pick a wrong row but never an out-of-range one
__device__ __forceinline__ int rg_find(const int64_t* __restrict__ off, int n, long long j) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= j) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// raw sample g of (s, c): the station's chunk block [r0, r1), the kept tail [r0 - min(W, r0), r0) before; 0.0f outside
__device__ __forceinline__ float rg_raw(const SeistRaggedStep& p, const float* tail, const float* chunk, int s, int c, long long r0,
                                        long long r1, long long g) {
  if (g >= r0)
    return g < r1 ? chunk[(size_t)p.C * p.chunk_off[s] + (size_t)c * (r1 - r0) + (size_t)(g - r0)] : 0.f;
  const long long h = g - (r0 - min((long long)p.W, r0));
  return h >= 0 ? tail[((size_t)s * p.C + c) * p.W + (size_t)h] : 0.f;
}

// x (B, C, W): row (b, c) = normalised window j0 + b of the call; zero from n_win on
__global__ void __launch_bounds__(PR_NT) ragged_window_kernel(SeistRaggedStep p, const float* __restrict__ tail,
                                                              const float* __restrict__ chunk, long long j0, float* __restrict__ x) {
  extern __shared__ float rw_row[];                 // [W]
  const int b = blockIdx.x / p.C, c = blockIdx.x % p.C;
  const long long j = j0 + b;
  float* dst = x + (size_t)blockIdx.x * p.W;
  if (j >= p.n_win) {
    for (int i = threadIdx.x; i < p.W; i += PR_NT) dst[i] = 0.f;
    return;
  }
  const int s = rg_find(p.win_off, p.S, j);
  const long long q = j - p.win_off[s], r0 = p.r0[s], r1 = p.r1[s];
  const long long a = q < p.nk[s] ? (p.k0[s] + q) * p.P : p.tail[s];
  for (int i = threadIdx.x; i < p.W; i += PR_NT) rw_row[i] = rg_raw(p, tail, chunk, s, c, r0, r1, a + i);
  __syncthreads();
  pr_normalize_row(rw_row, dst, p.W, p.norm_mode);
}

// stream_stack_kernel per station: CTA (x, s - s0, c) gathers the batch's windows of station s into its acc block
__global__ void __launch_bounds__(ST_NT) ragged_stack_kernel(SeistRaggedStep p, const float* __restrict__ y, long long j0, int nb, int s0,
                                                             const float* __restrict__ carry, float* __restrict__ acc) {
  const int s = s0 + blockIdx.y, c = blockIdx.z;
  if (s >= p.S) return;
  const long long wb = p.win_off[s], nw = p.win_off[s + 1] - wb;
  const long long qa = max(j0 - wb, 0LL), qb = min(j0 + nb - 1 - wb, nw - 1);
  if (qa > qb) return;
  const long long nk = p.nk[s], k0 = p.k0[s], tl0 = p.tail[s], f0 = p.f0[s], r1 = p.r1[s];
  const long long sa = qa < nk ? (k0 + qa) * p.P : tl0, sb = qb < nk ? (k0 + qb) * p.P : tl0;
  const long long t = sa + blockIdx.x * (long long)ST_NT + threadIdx.x;
  if (t >= sb + p.W || t < f0 || t >= r1) return;
  const long long lo = t < p.W ? 0 : (t - p.W) / p.P + 1, hi = min(t / p.P, k0 + nk - 1);
  const bool reg = lo <= hi;                                   // else the tail window is t's only one
  const bool tl = tl0 >= 0 && qb == nw - 1 && t >= tl0;
  const bool first = reg ? (qa < nk && lo >= k0 + qa) : tl;
  const long long L = r1 - f0;
  float* out = acc + (size_t)3 * p.acc_off[s] + (size_t)c * L + (size_t)(t - f0);
  float a = first ? (p.stack_mode == 0 ? 0.f : -INFINITY)
                  : (qa > 0 ? *out : (t - f0 < p.W ? carry[((size_t)s * 3 + c) * p.W + (size_t)(t - f0)] : 0.f));
  const float* yb = y + (size_t)c * p.W;
  const long long kb = min(hi, k0 + min(qb, nk - 1));
  for (long long k = max(lo, k0 + qa); k <= kb; ++k) {
    const float v = yb[(size_t)(wb + (k - k0) - j0) * 3 * p.W + (size_t)(t - k * p.P)];
    a = p.stack_mode == 0 ? a + v : fmaxf(a, v);
  }
  if (tl) {
    const float v = yb[(size_t)(wb + nk - j0) * 3 * p.W + (size_t)(t - tl0)];
    a = p.stack_mode == 0 ? a + v : fmaxf(a, v);
  }
  *out = a;
}

// CTA (x, s, c): probs block of s = final [f0, f1), carry_out = partial sums of [f1, r1), as stream_emit_kernel
__global__ void __launch_bounds__(ST_NT) ragged_emit_kernel(SeistRaggedStep p, const float* __restrict__ carry, const float* __restrict__ acc,
                                                            float* __restrict__ probs, float* __restrict__ carry_out) {
  const int s = blockIdx.y, c = blockIdx.z;
  const long long f0 = p.f0[s], r1 = p.r1[s], i = blockIdx.x * (long long)ST_NT + threadIdx.x;
  if (i >= r1 - f0) return;
  const long long t = f0 + i, f1 = p.f1[s], nk = p.nk[s], k0 = p.k0[s], tl0 = p.tail[s], kr = p.kr[s];
  const bool touched = (nk > 0 && t >= k0 * p.P && t < (k0 + nk - 1) * p.P + p.W) || (tl0 >= 0 && t >= tl0);
  const size_t row = (size_t)s * 3 + c;
  float v = touched ? acc[(size_t)3 * p.acc_off[s] + (size_t)c * (r1 - f0) + (size_t)i]
                    : (t < p.r0[s] && i < p.W ? carry[row * p.W + (size_t)i] : 0.f);   // t >= r0 untouched: no window yet
  if (t < f1) {
    if (p.stack_mode == 0) {
      const long long lo = t < p.W ? 0 : (t - p.W) / p.P + 1, hi = kr >= 0 ? min(t / p.P, kr - 1) : t / p.P;
      const int cnt = (int)max(hi - lo + 1, 0LL) + (tl0 >= 0 && t >= tl0 ? 1 : 0);
      v = __fdiv_rn(v, (float)cnt);
    }
    probs[(size_t)3 * p.out_off[s] + (size_t)c * (f1 - f0) + (size_t)i] = v;
  } else if (t - f1 < p.W) {
    carry_out[row * p.W + (size_t)(t - f1)] = v;
  }
}

// tail_out (S, C, W): the last min(W, r1[s]) raw samples of each station after the call
__global__ void __launch_bounds__(ST_NT) ragged_keep_kernel(SeistRaggedStep p, const float* __restrict__ tail,
                                                            const float* __restrict__ chunk, float* __restrict__ tail_out) {
  const int s = blockIdx.y / p.C, c = blockIdx.y % p.C;
  const long long r0 = p.r0[s], r1 = p.r1[s], keep = min((long long)p.W, r1);
  const int i = blockIdx.x * ST_NT + threadIdx.x;
  if (i < keep) tail_out[(size_t)blockIdx.y * p.W + i] = rg_raw(p, tail, chunk, s, c, r0, r1, r1 - keep + i);
}

// ---- raw histories of a ragged characterised stream (DESIGN §4.20) -------------------------------------------------
// Station s's history is a (C, len_s) block at C * off[s] of a packed buffer, len_s = off[s + 1] - off[s], its first
// sample the global h0[s].  CTA (x, s * C + c): out row (s, c) = samples [h0_out[s], h0_out[s] + n_out) of the held row
// (base h0_held[s]) followed by the station's chunk block; every read is range-checked against the station's own
// counts and the buffer's capacity (0.0f outside), every write against out's capacity.
__global__ void __launch_bounds__(ST_NT) ragged_history_kernel(const float* __restrict__ held, const long long* __restrict__ held_off,
                                                               const long long* __restrict__ h0_held, long long held_cap,
                                                               const float* __restrict__ chunk, const long long* __restrict__ chunk_off,
                                                               long long chunk_cap, const long long* __restrict__ h0_out,
                                                               const long long* __restrict__ out_off, int C, float* __restrict__ out,
                                                               long long out_cap) {
  const int s = blockIdx.y / C, c = blockIdx.y % C;
  const long long o0 = out_off[s], n_out = out_off[s + 1] - o0;
  const long long i = (long long)blockIdx.x * ST_NT + threadIdx.x;
  if (i >= n_out) return;
  const long long a0 = held_off[s], n_held = held_off[s + 1] - a0, b0 = chunk_off[s], n = chunk_off[s + 1] - b0;
  const long long j = h0_out[s] - h0_held[s] + i;
  const long long hi = C * a0 + c * n_held + j, ci = C * b0 + c * n + (j - n_held);
  float v = 0.f;
  if (j >= 0 && j < n_held && hi < held_cap) v = held[hi];
  else if (j >= n_held && j - n_held < n && ci < chunk_cap) v = chunk[ci];
  const long long w = C * o0 + c * n_out + i;
  if (w < out_cap) out[w] = v;
}

// event_windows_kernel cutting from packed histories: p = index[e0 + b] - h0[s] in station s's row, 0.0f outside
// [0, len_s); events >= M and picks outside the station's history give zero rows
__global__ void __launch_bounds__(PR_NT) ragged_event_windows_kernel(const float* __restrict__ hist, const long long* __restrict__ hist_off,
                                                                     const long long* __restrict__ h0, long long hist_cap, int S, int C,
                                                                     const long long* __restrict__ index,
                                                                     const long long* __restrict__ offsets, long long M, long long e0,
                                                                     int W, int a, int mode, EventDst dst, int n_dst) {
  extern __shared__ float rew_row[];                // [W]: the zero-filled history slice, normalised in place
  const int b = blockIdx.x / C, c = blockIdx.x % C;
  const long long e = e0 + b;
  const size_t row = (size_t)blockIdx.x * W;
  const int s = rg_find((const int64_t*)offsets, S, e);
  const long long h = hist_off[s], len = hist_off[s + 1] - h;
  const long long p = e < M ? index[e] - h0[s] : -1;
  if (p < 0 || p >= len) {
#pragma unroll
    for (int d = 0; d < EW_MAX_DST; ++d)
      if (d < n_dst)
        for (int i = threadIdx.x; i < W; i += PR_NT) dst.x[d][row + i] = 0.f;
    return;
  }
  const long long src = C * h + c * len, t0 = p - a;
  for (int i = threadIdx.x; i < W; i += PR_NT) {
    const long long t = t0 + i;
    rew_row[i] = t >= 0 && t < len && src + t < hist_cap ? hist[src + t] : 0.f;
  }
  __syncthreads();
  pr_normalize_row(rew_row, rew_row, W, mode);
#pragma unroll
  for (int d = 0; d < EW_MAX_DST; ++d)
    if (d < n_dst)
      for (int i = threadIdx.x; i < W; i += PR_NT) dst.x[d][row + i] = rew_row[i];
}

// ragged_event_windows_kernel for a gapped stream (DESIGN §4.23): event e is a pick of position q, the last with
// pos_off[q] <= e (a bounded search, always in [0, n_pos)); the position names its station and its segment's global
// [on, end].  Samples outside [on, end] ∩ [h0_s, R_s) read as 0.0f, so the window is that of segment_event_windows_kernel.
// A station outside [0, S), a pick outside its segment or its station's history, and events >= M give zero rows.
__global__ void __launch_bounds__(PR_NT) gap_event_windows_kernel(const float* __restrict__ hist, const long long* __restrict__ hist_off,
                                                                  const long long* __restrict__ h0, long long hist_cap, int S, int C,
                                                                  const long long* __restrict__ pos_station,
                                                                  const long long* __restrict__ pos_on, const long long* __restrict__ pos_end,
                                                                  const long long* __restrict__ pos_off, int n_pos,
                                                                  const long long* __restrict__ index, long long M, long long e0, int W,
                                                                  int a, int mode, EventDst dst, int n_dst) {
  extern __shared__ float gew_row[];                // [W]: the zero-filled segment slice of the history, normalised in place
  const int b = blockIdx.x / C, c = blockIdx.x % C;
  const long long e = e0 + b;
  const size_t row = (size_t)blockIdx.x * W;
  const int q = rg_find((const int64_t*)pos_off, n_pos, e);
  const long long s = pos_station[q];
  const bool in = e < M && s >= 0 && s < S;
  const long long hs = in ? hist_off[s] : 0, len = in ? hist_off[s + 1] - hs : 0, base = in ? h0[s] : 0;
  const long long lo = max(pos_on[q], base), hi = min(pos_end[q] + 1, base + len);   // readable: [lo, hi), global
  const long long p = in ? index[e] : -1;
  if (!in || p < lo || p >= hi) {
#pragma unroll
    for (int d = 0; d < EW_MAX_DST; ++d)
      if (d < n_dst)
        for (int i = threadIdx.x; i < W; i += PR_NT) dst.x[d][row + i] = 0.f;
    return;
  }
  const long long src = C * hs + c * len - base, t0 = p - a;
  for (int i = threadIdx.x; i < W; i += PR_NT) {
    const long long t = t0 + i;
    gew_row[i] = t >= lo && t < hi && src + t >= 0 && src + t < hist_cap ? hist[src + t] : 0.f;
  }
  __syncthreads();
  pr_normalize_row(gew_row, gew_row, W, mode);
#pragma unroll
  for (int d = 0; d < EW_MAX_DST; ++d)
    if (d < n_dst)
      for (int i = threadIdx.x; i < W; i += PR_NT) dst.x[d][row + i] = gew_row[i];
}

// channel ch of row s of a packed ext, and its length
__device__ __forceinline__ const float* rg_row(const float* ext, const long long* __restrict__ ext_off, int C, int ch, int s, long long& L) {
  const long long e0 = ext_off[s];
  L = ext_off[s + 1] - e0;
  return ext + (size_t)C * e0 + (size_t)ch * L;
}

// CTA (x, s, c): ext row = look, the stretch, -inf; look_out = its samples m, m + 1
__global__ void __launch_bounds__(ST_NT) ragged_ext_kernel(const float* __restrict__ look, const float* __restrict__ probs,
                                                           const long long* __restrict__ prob_off, const long long* __restrict__ ext_off,
                                                           int C, float* __restrict__ ext, float* __restrict__ look_out) {
  const int s = blockIdx.y, c = blockIdx.z;
  const long long e0 = ext_off[s], L = ext_off[s + 1] - e0, p0 = prob_off[s], m = prob_off[s + 1] - p0;
  const long long i = blockIdx.x * (long long)ST_NT + threadIdx.x;
  if (i >= L) return;
  const float v = i < 2 ? look[((size_t)s * C + c) * 2 + i] : (i - 2 < m ? probs[(size_t)C * p0 + (size_t)c * m + (size_t)(i - 2)] : -INFINITY);
  ext[(size_t)C * e0 + (size_t)c * L + (size_t)i] = v;
  if (i == m || i == m + 1) look_out[((size_t)s * C + c) * 2 + (size_t)(i - m)] = v;
}

// pending candidates of the previous call ([nclosed, ncand) of its rows) to the front of this call's rows, rebased by
// -delta[s]
__global__ void __launch_bounds__(ST_NT) rg_pend_move_kernel(const int* __restrict__ pci, const float* __restrict__ pcv, int pcapc,
                                                             const int* __restrict__ pnclosed, const int* __restrict__ pncand,
                                                             const long long* __restrict__ delta, int* __restrict__ cidx,
                                                             float* __restrict__ cval, int capc, int* __restrict__ npend) {
  const int s = blockIdx.y;
  const int a = pci ? pnclosed[s] : 0, m = pci ? pncand[s] - a : 0;
  if (blockIdx.x == 0 && threadIdx.x == 0) npend[s] = m;
  if (m == 0) return;
  const long long d = delta[s];
  for (int j = blockIdx.x * ST_NT + threadIdx.x; j < m; j += gridDim.x * ST_NT) {
    cidx[(size_t)s * capc + j] = (int)(pci[(size_t)s * pcapc + a + j] - d);
    cval[(size_t)s * capc + j] = pcv[(size_t)s * pcapc + a + j];
  }
}

// the tested range of a row: [max(lo, 1), min(hi, L - 2)]
__device__ __forceinline__ void rg_range(const long long* lo_a, const long long* hi_a, int s, long long L, long long lim_hi, long long& lo,
                                         long long& hi) {
  lo = max(lo_a[s], 1LL);
  hi = min(hi_a[s], L - lim_hi);
}

// cand_count_kernel over each row's own range; blocks past it count 0
__global__ void __launch_bounds__(ST_NT) rg_cand_count_kernel(const float* __restrict__ ext, const long long* __restrict__ ext_off, int C,
                                                              int ch, const long long* __restrict__ lo_a, const long long* __restrict__ hi_a,
                                                              float mph, int* __restrict__ blk, int nblk) {
  __shared__ int warp_s[ST_NT / 32];
  long long L, lo, hi;
  const float* x = rg_row(ext, ext_off, C, ch, blockIdx.y, L);
  rg_range(lo_a, hi_a, blockIdx.y, L, 2, lo, hi);
  const long long a = lo + (long long)blockIdx.x * ST_CH;
  int n = 0;
  for (long long i = a + threadIdx.x; i < min(a + ST_CH, hi + 1); i += ST_NT) n += pk_cand(x, (int)i, mph);
  n = st_block_count(n, warp_s);
  if (threadIdx.x == 0) blk[(size_t)blockIdx.y * nblk + blockIdx.x] = n;
}

// cand_fill_kernel with a per-row index shift, behind the row's pending candidates
__global__ void __launch_bounds__(ST_NT) rg_cand_fill_kernel(const float* __restrict__ ext, const long long* __restrict__ ext_off, int C,
                                                             int ch, const long long* __restrict__ lo_a, const long long* __restrict__ hi_a,
                                                             float mph, const int* __restrict__ blk, int nblk, const int* __restrict__ off0,
                                                             const long long* __restrict__ ishift, int capc, int* __restrict__ cidx,
                                                             float* __restrict__ cval) {
  __shared__ int warp_s[ST_NT / 32];
  const int s = blockIdx.y;
  long long L, lo, hi;
  const float* x = rg_row(ext, ext_off, C, ch, s, L);
  rg_range(lo_a, hi_a, s, L, 2, lo, hi);
  const long long a = lo + (long long)blockIdx.x * ST_CH;
  if (a > hi) return;                                          // the whole CTA: past the row's range
  const int sh = (int)ishift[s];
  int base = blk[(size_t)s * nblk + blockIdx.x] + off0[s];
  int* ci = cidx + (size_t)s * capc;
  float* cv = cval + (size_t)s * capc;
  for (long long i0 = a; i0 < min(a + ST_CH, hi + 1); i0 += ST_NT) {
    const long long i = i0 + threadIdx.x;
    const bool f = i <= hi && pk_cand(x, (int)i, mph);
    int tot;
    const int r = st_block_rank(f, warp_s, tot);
    if (f && base + r < capc) { ci[base + r] = (int)i + sh; cv[base + r] = x[i]; }
    base += tot;
  }
}

// per row: ncand = pending + new; the closed prefix ends before the last cluster unless its last candidate c has
// c + mpd <= lim[s] (no later candidate can join it); info = (pending count, global index of the first pending one)
__global__ void __launch_bounds__(ST_NT) rg_close_scan_kernel(const int* __restrict__ npend, const int* __restrict__ nnew,
                                                              const int* __restrict__ cidx, int capc, int mpd,
                                                              const long long* __restrict__ lim_a, const long long* __restrict__ base_a,
                                                              int* __restrict__ ncand, int* __restrict__ nclosed, long long* __restrict__ info) {
  __shared__ int last_s;
  const int s = blockIdx.x, n = min(npend[s] + nnew[s], capc);
  const int* ci = cidx + (size_t)s * capc;
  if (threadIdx.x == 0) last_s = 0;
  __syncthreads();
  for (int top = n - 1; top >= 1; top -= ST_NT) {            // the last cluster start, searched from the end
    const int j = top - (int)threadIdx.x;
    const bool f = j >= 1 && ci[j] - ci[j - 1] > mpd;
    if (f) atomicMax(&last_s, j);
    if (__syncthreads_or(f)) break;
  }
  if (threadIdx.x == 0) {
    const int nc = n == 0 || (long long)ci[n - 1] + mpd <= lim_a[s] ? n : last_s;
    ncand[s] = n;
    nclosed[s] = nc;
    info[s] = n - nc;
    info[gridDim.x + s] = nc < n ? base_a[s] + ci[nc] : LLONG_MAX;
  }
}

// keep_fill_kernel with the index base per row
__global__ void __launch_bounds__(ST_NT) rg_keep_fill_kernel(const int* __restrict__ ncand, int capc, const int* __restrict__ cidx,
                                                             const float* __restrict__ cval, const unsigned char* __restrict__ state,
                                                             const int* __restrict__ blk, int nblk, const long long* __restrict__ offsets,
                                                             const long long* __restrict__ base_a, long long* __restrict__ index,
                                                             float* __restrict__ value) {
  __shared__ int warp_s[ST_NT / 32];
  const int n = ncand[blockIdx.y];
  const int a = blockIdx.x * ST_CH;
  if (a >= n) return;
  const size_t r0 = (size_t)blockIdx.y * capc;
  const long long sh = base_a[blockIdx.y];
  long long b = offsets[blockIdx.y] + blk[(size_t)blockIdx.y * nblk + blockIdx.x];
  for (int j0 = a; j0 < min(a + ST_CH, n); j0 += ST_NT) {
    const int j = j0 + threadIdx.x;
    const bool f = j < n && state[r0 + j] == CL_KEEP;
    int tot;
    const int r = st_block_rank(f, warp_s, tot);
    if (f) { index[b + r] = cidx[r0 + j] + sh; value[b + r] = cval[r0 + j]; }
    b += tot;
  }
}

// the run ends in each row's own range [max(lo, 1), min(hi, L - 1)], per block; open_out = the open run carried past it
__global__ void __launch_bounds__(ST_NT) rg_srun_count_kernel(const float* __restrict__ ext, const long long* __restrict__ ext_off, int C,
                                                              int ch, const long long* __restrict__ lo_a, const long long* __restrict__ hi_a,
                                                              float thr, int* __restrict__ blk, int nblk, const long long* __restrict__ open_in,
                                                              long long* __restrict__ open_out) {
  __shared__ int warp_s[ST_NT / 32];
  long long L, lo, hi;
  const float* x = rg_row(ext, ext_off, C, ch, blockIdx.y, L);
  rg_range(lo_a, hi_a, blockIdx.y, L, 1, lo, hi);
  hi = max(hi, lo - 1);
  const long long a = lo + (long long)blockIdx.x * ST_CH;
  int n = 0;
  for (long long i = a + threadIdx.x; i < min(a + ST_CH, hi + 1); i += ST_NT) n += sr_off(x, (int)i, thr);
  n = st_block_count(n, warp_s);
  if (threadIdx.x == 0) {
    blk[(size_t)blockIdx.y * nblk + blockIdx.x] = n;
    if (blockIdx.x == 0) open_out[blockIdx.y] = x[hi] > thr ? open_in[blockIdx.y] : -1;   // raised by the fill on a new start
  }
}

// blk: exclusive counts of run ends before each block.  The run ending at the k-th end of row s is pair offsets[s] + k;
// the carried open run is the first of them.  Pairs are global (g0[s] + position).
__global__ void __launch_bounds__(ST_NT) rg_srun_fill_kernel(const float* __restrict__ ext, const long long* __restrict__ ext_off, int C,
                                                             int ch, const long long* __restrict__ lo_a, const long long* __restrict__ hi_a,
                                                             float thr, const long long* __restrict__ g0_a, const int* __restrict__ blk,
                                                             int nblk, const long long* __restrict__ offsets,
                                                             const long long* __restrict__ open_in, long long* __restrict__ open_out,
                                                             long long* __restrict__ pairs) {
  __shared__ int warp_s[ST_NT / 32];
  const int s = blockIdx.y;
  long long L, lo, hi;
  const float* x = rg_row(ext, ext_off, C, ch, s, L);
  rg_range(lo_a, hi_a, s, L, 1, lo, hi);
  hi = max(hi, lo - 1);
  const long long end = offsets[s + 1];
  if (blockIdx.x == 0 && threadIdx.x == 0 && open_in[s] >= 0 && end > offsets[s]) pairs[offsets[s] * 2] = open_in[s];
  const long long a = lo + (long long)blockIdx.x * ST_CH;
  if (a > hi) return;                                          // the whole CTA: past the row's range
  const long long g0 = g0_a[s];
  const bool open_end = x[hi] > thr;
  long long off_base = offsets[s] + blk[(size_t)s * nblk + blockIdx.x];
  long long on_base = off_base + (x[a - 1] > thr ? 1 : 0);    // a run open into the block ends before the next starts
  for (long long i0 = a; i0 < min(a + ST_CH, hi + 1); i0 += ST_NT) {
    const long long i = i0 + threadIdx.x;
    const bool fon = i <= hi && sr_on(x, (int)i, thr), foff = i <= hi && sr_off(x, (int)i, thr);
    int ton, toff;
    const int ron = st_block_rank(fon, warp_s, ton);
    const int roff = st_block_rank(foff, warp_s, toff);
    if (foff) pairs[(off_base + roff) * 2 + 1] = g0 + i - 1;
    if (fon) {
      if (on_base + ron < end) pairs[(on_base + ron) * 2] = g0 + i;
      else if (open_end) atomicMax(&open_out[s], g0 + i);
    }
    on_base += ton;
    off_base += toff;
  }
}

// ---- whole records with data gaps (DESIGN §4.21) --------------------------------------------------------------------
// A sample is usable when every channel is finite; a segment is a maximal run of usable samples.  Each thread tests its
// own sample and takes its neighbour's verdict from the next lane, so a pass reads every sample of the record once.
__device__ __forceinline__ bool gp_ok(const float* x, int C, long long T, long long t) {
  bool ok = true;
  for (int c = 0; c < C; ++c) ok = ok && isfinite(x[(size_t)c * T + t]);
  return ok;
}

// the segment starts of block blockIdx.x (ST_CH samples) of the row x (C, T): the CTA's count
__device__ __forceinline__ int gp_count_block(const float* x, int C, int T, int* warp_s) {
  const int a = blockIdx.x * ST_CH, e = min(a + ST_CH, T), lane = threadIdx.x & 31;
  int n = 0;
  for (int i0 = a; i0 < e; i0 += ST_NT) {
    const int i = i0 + threadIdx.x;
    const bool ok = i < e && gp_ok(x, C, T, i);
    bool prev = __shfl_up_sync(0xffffffffu, ok, 1);
    if (lane == 0) prev = i > 0 && i < e && gp_ok(x, C, T, i - 1);
    n += ok && !prev;
  }
  return st_block_count(n, warp_s);
}

// blocks of ST_CH samples; blk (S, nblk): the segment starts of each block
__global__ void __launch_bounds__(ST_NT) gap_count_kernel(const float* __restrict__ rec, int C, int T, int* __restrict__ blk, int nblk) {
  __shared__ int warp_s[ST_NT / 32];
  const int n = gp_count_block(rec + (size_t)blockIdx.y * C * T, C, T, warp_s);
  if (threadIdx.x == 0) blk[(size_t)blockIdx.y * nblk + blockIdx.x] = n;
}

// the [on, off] of the segments of block blockIdx.x of the row x (C, T), the block's first start at table row b0
__device__ __forceinline__ void gp_fill_block(const float* x, int C, int T, long long b0, long long cap, long long* pairs, int* warp_s) {
  const int a = blockIdx.x * ST_CH, e = min(a + ST_CH, T), lane = threadIdx.x & 31;
  long long on_base = b0, off_base = b0 - (a > 0 && gp_ok(x, C, T, a - 1) && gp_ok(x, C, T, a) ? 1 : 0);
  for (int i0 = a; i0 < e; i0 += ST_NT) {
    const int i = i0 + threadIdx.x;
    const bool ok = i < e && gp_ok(x, C, T, i);
    bool prev = __shfl_up_sync(0xffffffffu, ok, 1), next = __shfl_down_sync(0xffffffffu, ok, 1);
    if (lane == 0) prev = i > 0 && i < e && gp_ok(x, C, T, i - 1);
    if (lane == 31) next = i + 1 < T && gp_ok(x, C, T, i + 1);   // i + 1 < e for every other lane of a full warp
    const bool fon = ok && !prev, foff = ok && (i == T - 1 || !next);
    int ton, toff;
    const int ron = st_block_rank(fon, warp_s, ton);
    const int roff = st_block_rank(foff, warp_s, toff);
    if (fon && on_base + ron < cap) pairs[(on_base + ron) * 2] = i;
    if (foff && off_base + roff >= 0 && off_base + roff < cap) pairs[(off_base + roff) * 2 + 1] = i;
    on_base += ton;
    off_base += toff;
  }
}

// run_fill_kernel with usable / not usable for p > thr: blk holds the exclusive start offsets per block, the ends before a
// block are as many, less one when a segment crosses into it; rows >= cap are dropped
__global__ void __launch_bounds__(ST_NT) gap_fill_kernel(const float* __restrict__ rec, int C, int T, const int* __restrict__ blk,
                                                         int nblk, const long long* __restrict__ offsets, long long cap,
                                                         long long* __restrict__ pairs) {
  __shared__ int warp_s[ST_NT / 32];
  const long long b0 = offsets[blockIdx.y] + blk[(size_t)blockIdx.y * nblk + blockIdx.x];
  gp_fill_block(rec + (size_t)blockIdx.y * C * T, C, T, b0, cap, pairs, warp_s);
}

// ---- streams with data gaps (DESIGN §4.22) --------------------------------------------------------------------------
// Station s's pushed samples are a (C, n_s) block at C * chunk_off[s] of a packed chunk of chunk_cap floats; a station
// whose block does not fit the chunk is read as empty.  The scan is gap_count / gap_fill per block; its table holds
// each segment's [on, off] in the station's block.
__device__ __forceinline__ bool gs_block(const long long* chunk_off, long long chunk_cap, int C, int s, long long& b, int& n) {
  b = chunk_off[s];
  const long long len = chunk_off[s + 1] - b;
  n = (int)len;
  return b >= 0 && len >= 0 && len <= INT32_MAX && C * (b + len) <= chunk_cap;
}

__global__ void __launch_bounds__(ST_NT) gap_stream_count_kernel(const float* __restrict__ chunk, long long chunk_cap,
                                                                 const long long* __restrict__ chunk_off, int C, int* __restrict__ blk,
                                                                 int nblk) {
  __shared__ int warp_s[ST_NT / 32];
  long long b;
  int n;
  if (!gs_block(chunk_off, chunk_cap, C, blockIdx.y, b, n)) b = n = 0;
  const int cnt = gp_count_block(chunk + C * b, C, n, warp_s);
  if (threadIdx.x == 0) blk[(size_t)blockIdx.y * nblk + blockIdx.x] = cnt;
}

__global__ void __launch_bounds__(ST_NT) gap_stream_fill_kernel(const float* __restrict__ chunk, long long chunk_cap,
                                                                const long long* __restrict__ chunk_off, int C, const int* __restrict__ blk,
                                                                int nblk, const long long* __restrict__ offsets, long long cap,
                                                                long long* __restrict__ pairs) {
  __shared__ int warp_s[ST_NT / 32];
  long long b;
  int n;
  if (!gs_block(chunk_off, chunk_cap, C, blockIdx.y, b, n) || (long long)blockIdx.x * ST_CH >= n) return;   // uniform per CTA
  const long long b0 = offsets[blockIdx.y] + blk[(size_t)blockIdx.y * nblk + blockIdx.x];
  gp_fill_block(chunk + C * b, C, n, b0, cap, pairs, warp_s);
}

// out row r (a (C, n_r) block at C * row_off[r], n_r = row_off[r + 1] - row_off[r]) = samples row_start[r] .. + n_r - 1
// of station row_station[r]'s block; 0.0f where the row reaches outside that block
__global__ void __launch_bounds__(ST_NT) gap_stream_pack_kernel(const float* __restrict__ chunk, long long chunk_cap,
                                                                const long long* __restrict__ chunk_off, int S, int C,
                                                                const long long* __restrict__ row_station,
                                                                const long long* __restrict__ row_start,
                                                                const long long* __restrict__ row_off, int n_rows, long long n,
                                                                float* __restrict__ out, long long out_cap) {
  for (long long e = blockIdx.x * (long long)ST_NT + threadIdx.x; e < n && e < out_cap; e += (long long)gridDim.x * ST_NT) {
    const int r = rg_find((const int64_t*)row_off, n_rows, e / C);
    const long long m = row_off[r + 1] - row_off[r], i = e - C * row_off[r];
    float v = 0.f;
    const long long st = row_station[r];
    if (m > 0 && i >= 0 && i < C * m && st >= 0 && st < S) {
      long long b;
      int ns;
      const long long c = i / m, t = row_start[r] + (i - c * m);
      if (gs_block(chunk_off, chunk_cap, C, (int)st, b, ns) && t >= 0 && t < ns) v = chunk[C * b + c * ns + t];
    }
    out[e] = v;
  }
}

// dst[dst_base[r] + c * dst_ld[r] + t] = src[src_base[r] + c * src_ld[r] + t] for c < 3, t < m_r = m_off[r + 1] - m_off[r];
// reads past src_cap give NaN, writes past dst_cap are dropped
__global__ void __launch_bounds__(ST_NT) gap_stream_copy_kernel(const float* __restrict__ src, long long src_cap,
                                                                const long long* __restrict__ m_off, const long long* __restrict__ src_base,
                                                                const long long* __restrict__ src_ld, const long long* __restrict__ dst_base,
                                                                const long long* __restrict__ dst_ld, int n_rows, long long n,
                                                                float* __restrict__ dst, long long dst_cap) {
  for (long long e = blockIdx.x * (long long)ST_NT + threadIdx.x; e < n; e += (long long)gridDim.x * ST_NT) {
    const int r = rg_find((const int64_t*)m_off, n_rows, e / 3);
    const long long m = m_off[r + 1] - m_off[r], i = e - 3 * m_off[r];
    if (m <= 0 || i < 0 || i >= 3 * m) continue;
    const long long c = i / m, t = i - c * m;
    const long long si = src_base[r] + c * src_ld[r] + t, di = dst_base[r] + c * dst_ld[r] + t;
    if (di >= 0 && di < dst_cap) dst[di] = si >= 0 && si < src_cap ? src[si] : NAN;
  }
}

// segment g of a table of G: its first sample, length and station when they describe an annotated segment of a record
// (S, ., T) for windows of W, else false
__device__ __forceinline__ bool sg_get(const long long* pairs, const long long* station, int G, int g, int S, long long T, int W,
                                       long long& on, long long& len, int& s) {
  if (g < 0 || g >= G) return false;
  on = pairs[2 * (size_t)g];
  len = pairs[2 * (size_t)g + 1] - on + 1;
  const long long st = station[g];
  s = (int)st;
  return on >= 0 && len >= W && on + len <= T && st >= 0 && st < S;
}

// the segment of station s holding sample t: the last g in the station's range with on_g <= t, when t <= off_g; else -1
__device__ __forceinline__ int sg_find(const long long* pairs, const long long* seg_off, int G, int s, long long t) {
  const long long g0 = min(max(seg_off[s], 0LL), (long long)G), g1 = min(max(seg_off[s + 1], g0), (long long)G);
  if (g0 >= g1 || pairs[2 * g0] > t) return -1;
  long long lo = g0, hi = g1 - 1;
  while (lo < hi) {
    const long long mid = (lo + hi + 1) >> 1;
    if (pairs[2 * mid] <= t) lo = mid; else hi = mid - 1;
  }
  return t <= pairs[2 * lo + 1] ? (int)lo : -1;
}

// x (B, C, W): row (b, c) = normalised record[s, c, on + start(q) : + W] for packed window j0 + b = window q of segment g
__global__ void __launch_bounds__(PR_NT) segment_window_kernel(const float* __restrict__ rec, int S, int C, long long T,
                                                               const long long* __restrict__ pairs, const long long* __restrict__ station,
                                                               const long long* __restrict__ win_off, int G, long long n_win, int W,
                                                               int P, long long j0, int mode, float* __restrict__ x) {
  extern __shared__ float sg_row[];                 // [W]: the record slice, read from global memory once
  const int b = blockIdx.x / C, c = blockIdx.x % C;
  const long long j = j0 + b;
  float* dst = x + (size_t)blockIdx.x * W;
  long long a = -1, on, len;
  int s = 0;
  if (j < n_win) {
    const int g = rg_find((const int64_t*)win_off, G, j);
    const long long q = j - win_off[g];
    if (sg_get(pairs, station, G, g, S, T, W, on, len, s) && q >= 0) {
      const Windows win((int)len, W, P);
      if (q < win.K) a = on + win.start((int)q);
    }
  }
  if (a < 0) {
    for (int i = threadIdx.x; i < W; i += PR_NT) dst[i] = 0.f;
    return;
  }
  const float* src = rec + ((size_t)s * C + c) * T + a;
  for (int i = threadIdx.x; i < W; i += PR_NT) sg_row[i] = src[i];
  __syncthreads();
  pr_normalize_row(sg_row, dst, W, mode);
}

// stack_batch_kernel per segment: CTA (x, g - g0, c) gathers the batch's windows of segment g into probs[s, c, on + t]
__global__ void __launch_bounds__(ST_NT) segment_stack_kernel(const float* __restrict__ y, int S, long long T,
                                                              const long long* __restrict__ pairs, const long long* __restrict__ station,
                                                              const long long* __restrict__ win_off, int G, int W, int P, long long j0,
                                                              int nb, int g0, int mode, float* __restrict__ probs) {
  const int g = g0 + blockIdx.y, c = blockIdx.z;
  long long on, len;
  int s;
  if (!sg_get(pairs, station, G, g, S, T, W, on, len, s)) return;
  const Windows win((int)len, W, P);
  const long long wb = win_off[g];
  const long long ka_ = max(j0 - wb, 0LL), kb_ = min(min(j0 + nb - 1 - wb, (long long)win.K - 1), win_off[g + 1] - wb - 1);
  if (ka_ > kb_) return;
  const int ka = (int)ka_, kb = (int)kb_;
  const int t = win.start(ka) + blockIdx.x * ST_NT + threadIdx.x;
  if (t >= win.start(kb) + W) return;
  int lo, hi;
  bool tail;
  win.cover(t, lo, hi, tail);
  const int first = lo <= hi ? lo : win.K - 1;
  float* out = probs + ((size_t)s * 3 + c) * T + on + t;
  float acc = first >= ka ? (mode == 0 ? 0.f : -INFINITY) : *out;
  const float* yb = y + (size_t)c * W;
  for (int k = max(lo, ka); k <= min(hi, kb); ++k) {
    const float v = yb[(size_t)(wb + k - j0) * 3 * W + (t - k * P)];
    acc = mode == 0 ? acc + v : fmaxf(acc, v);
  }
  if (tail && win.K - 1 >= ka && win.K - 1 <= kb) {
    const float v = yb[(size_t)(wb + win.K - 1 - j0) * 3 * W + (t - (win.T - W))];
    acc = mode == 0 ? acc + v : fmaxf(acc, v);
  }
  *out = acc;
}

// mean: one IEEE division by the covering windows within the segment; NaN outside every annotated segment
__global__ void __launch_bounds__(ST_NT) segment_finish_kernel(float* __restrict__ probs, int S, long long T,
                                                               const long long* __restrict__ pairs, const long long* __restrict__ seg_off,
                                                               int G, int W, int P, int mode, long long n) {
  for (long long i = blockIdx.x * (long long)ST_NT + threadIdx.x; i < n; i += (long long)gridDim.x * ST_NT) {
    const int s = (int)(i / (3 * T));
    const long long t = i % T;
    const int g = sg_find(pairs, seg_off, G, s, t);
    const long long on = g >= 0 ? pairs[2 * (size_t)g] : 0, len = g >= 0 ? pairs[2 * (size_t)g + 1] - on + 1 : 0;
    if (g < 0 || len < W || on < 0 || on + len > T) {
      probs[i] = NAN;
    } else if (mode == 0) {
      int lo, hi;
      bool tail;
      Windows((int)len, W, P).cover((int)(t - on), lo, hi, tail);
      const int cnt = max(hi - lo + 1, 0) + (tail ? 1 : 0);
      probs[i] = __fdiv_rn(probs[i], (float)cnt);
    }
  }
}

// CTA (x, r, c): flat (3, m_r) block of row r at 3 * prob_off[r] = probs[s, c, on + i] of segment rows[r] (0.0f when the
// row names no segment of the table or runs past the record)
__global__ void __launch_bounds__(ST_NT) segment_gather_kernel(const float* __restrict__ probs, int S, long long T,
                                                               const long long* __restrict__ pairs, const long long* __restrict__ station,
                                                               int G, const long long* __restrict__ rows,
                                                               const long long* __restrict__ prob_off, long long cap,
                                                               float* __restrict__ flat) {
  const int r = blockIdx.y, c = blockIdx.z;
  const long long o0 = prob_off[r], m = prob_off[r + 1] - o0, i = blockIdx.x * (long long)ST_NT + threadIdx.x;
  if (i >= m) return;
  const long long g = rows[r];
  float v = 0.f;
  if (g >= 0 && g < G) {
    const long long on = pairs[2 * g], st = station[g];
    if (st >= 0 && st < S && on >= 0 && on + i < T) v = probs[((size_t)st * 3 + c) * T + on + i];
  }
  const long long w = 3 * o0 + c * m + i;
  if (w >= 0 && w < cap) flat[w] = v;
}

// event_windows_kernel zero-filling outside the pick's own annotated segment [on, off]; picks outside every annotated
// segment give zero rows
__global__ void __launch_bounds__(PR_NT) segment_event_windows_kernel(const float* __restrict__ rec, int S, int C, long long T,
                                                                      const long long* __restrict__ pairs,
                                                                      const long long* __restrict__ seg_off,
                                                                      const unsigned char* __restrict__ annotated, int G,
                                                                      const long long* __restrict__ index,
                                                                      const long long* __restrict__ offsets, long long M, long long e0,
                                                                      int W, int a, int mode, EventDst dst, int n_dst) {
  extern __shared__ float sew_row[];                // [W]: the zero-filled segment slice, normalised in place
  const int b = blockIdx.x / C, c = blockIdx.x % C;
  const long long e = e0 + b;
  const size_t row = (size_t)blockIdx.x * W;
  const long long p = e < M ? index[e] : -1;
  const int s = rg_find((const int64_t*)offsets, S, e);
  const int g = p >= 0 && p < T ? sg_find(pairs, seg_off, G, s, p) : -1;
  const long long on = g >= 0 ? pairs[2 * (size_t)g] : 0, off = g >= 0 ? pairs[2 * (size_t)g + 1] : -1;
  if (g < 0 || !annotated[g] || on < 0 || off >= T) {
#pragma unroll
    for (int d = 0; d < EW_MAX_DST; ++d)
      if (d < n_dst)
        for (int i = threadIdx.x; i < W; i += PR_NT) dst.x[d][row + i] = 0.f;
    return;
  }
  const float* src = rec + ((size_t)s * C + c) * T;
  const long long t0 = p - a;
  for (int i = threadIdx.x; i < W; i += PR_NT) {
    const long long t = t0 + i;
    sew_row[i] = t >= on && t <= off ? src[t] : 0.f;
  }
  __syncthreads();
  pr_normalize_row(sew_row, sew_row, W, mode);
#pragma unroll
  for (int d = 0; d < EW_MAX_DST; ++d)
    if (d < n_dst)
      for (int i = threadIdx.x; i < W; i += PR_NT) dst.x[d][row + i] = sew_row[i];
}

// ---- work buffers ---------------------------------------------------------------------------------------------------
__host__ __device__ inline size_t st_align(size_t b) { return (b + 255) & ~(size_t)255; }
inline int st_capc(int T) { return T / 2 + 1; }                 // candidates of a row: never two adjacent samples
inline int st_nblk(int n) { return (n + ST_CH - 1) / ST_CH; }

struct PeakWork {
  int* ncand;
  int* nkeep;
  int* blk;
  int* cidx;
  float* cval;
  unsigned char* state;
  size_t bytes;
  PeakWork(void* base, int R, int T) {
    char* p = (char*)base;
    const size_t capc = st_capc(T);
    size_t o = 0;
    ncand = (int*)(p + o);            o += st_align(sizeof(int) * R);
    nkeep = (int*)(p + o);            o += st_align(sizeof(int) * R);
    blk = (int*)(p + o);              o += st_align(sizeof(int) * (size_t)R * st_nblk(T));
    cidx = (int*)(p + o);             o += st_align(sizeof(int) * (size_t)R * capc);
    cval = (float*)(p + o);           o += st_align(sizeof(float) * (size_t)R * capc);
    state = (unsigned char*)(p + o);  o += st_align((size_t)R * capc);
    bytes = o;
  }
};

struct StreamPeakWork {
  int* npend;
  int* nnew;
  int* ncand;
  int* nclosed;
  int* nkeep;
  int* blk;
  int* cidx;
  float* cval;
  unsigned char* state;
  int nblk;
  size_t bytes;
  StreamPeakWork(const void* base, int R, int capc, long long L) {
    char* p = (char*)base;
    nblk = std::max(st_nblk((int)L), st_nblk(capc));
    size_t o = 0;
    npend = (int*)(p + o);            o += st_align(sizeof(int) * R);
    nnew = (int*)(p + o);             o += st_align(sizeof(int) * R);
    ncand = (int*)(p + o);            o += st_align(sizeof(int) * R);
    nclosed = (int*)(p + o);          o += st_align(sizeof(int) * R);
    nkeep = (int*)(p + o);            o += st_align(sizeof(int) * R);
    blk = (int*)(p + o);              o += st_align(sizeof(int) * (size_t)R * nblk);
    cidx = (int*)(p + o);             o += st_align(sizeof(int) * (size_t)R * capc);
    cval = (float*)(p + o);           o += st_align(sizeof(float) * (size_t)R * capc);
    state = (unsigned char*)(p + o);  o += st_align((size_t)R * capc);
    bytes = o;
  }
};

inline size_t run_work_bytes(int R, int T) { return st_align(sizeof(int) * R) + st_align(sizeof(int) * (size_t)R * st_nblk(T)); }

}  // namespace seist

using namespace seist;

extern "C" {

int seist_window_batch(const float* record, int32_t S, int32_t C, int64_t T, int32_t W, int32_t P, int64_t w0, int32_t B,
                       int32_t mode, float* x, void* stream) {
  if (!record || !x || S <= 0 || C <= 0 || W < 1 || W > 49152 || T < W || T > INT32_MAX || P < 1 || P > W || w0 < 0 || B <= 0 ||
      mode < 0 || mode > 2) {
    set_error("window_batch: bad arguments (W <= T < 2^31, 1 <= W <= 49152, 1 <= P <= W, mode 0 none, 1 std, 2 max)");
    return -1;
  }
  static int attr = 0;
  const int smem = (int)sizeof(float) * W;
  if (smem > 48 * 1024 && smem > attr) {
    cudaFuncSetAttribute(window_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr = smem;
  }
  window_batch_kernel<<<(unsigned)((long long)B * C), PR_NT, smem, (cudaStream_t)stream>>>(record, S, C, Windows((int)T, W, P), w0,
                                                                                           mode, x);
  note_launch();
  return check_launch("window_batch");
}

int seist_event_windows(const float* record, int32_t S, int32_t C, int64_t T, const int64_t* index, int64_t M,
                        const int64_t* offsets, int64_t e0, int32_t B, int32_t W, int32_t anchor, int32_t mode, float* const* x,
                        int32_t n_dst, void* stream) {
  bool ok = record && (index || M == 0) && offsets && x && S > 0 && C > 0 && T >= 1 && T <= INT32_MAX && M >= 0 && e0 >= 0 && B > 0 &&
            (long long)B * C <= INT32_MAX && W >= 1 && W <= 49152 && anchor >= 0 && anchor <= W && mode >= 0 && mode <= 2 &&
            n_dst >= 1 && n_dst <= EW_MAX_DST;
  EventDst dst{};
  for (int d = 0; ok && d < n_dst; ++d) ok = (dst.x[d] = x[d]) != nullptr;
  if (!ok) {
    set_error("event_windows: bad arguments (1 <= T < 2^31, 1 <= W <= 49152, 0 <= anchor <= W, M >= 0, e0 >= 0, B > 0, "
              "mode 0 none, 1 std, 2 max, 1 to 4 non-null destinations)");
    return -1;
  }
  static int attr = 0;
  const int smem = (int)sizeof(float) * W;
  if (smem > 48 * 1024 && smem > attr) {
    cudaFuncSetAttribute(event_windows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr = smem;
  }
  event_windows_kernel<<<(unsigned)((long long)B * C), PR_NT, smem, (cudaStream_t)stream>>>(
      record, S, C, (int)T, (const long long*)index, (const long long*)offsets, M, e0, W, anchor, mode, dst, n_dst);
  note_launch();
  return check_launch("event_windows");
}

int seist_stack_batch(const float* y, int32_t S, int64_t T, int32_t W, int32_t P, int64_t w0, int32_t B, int32_t mode, float* probs,
                      void* stream) {
  if (!y || !probs || S <= 0 || W < 1 || T < W || T > INT32_MAX || P < 1 || P > W || w0 < 0 || B <= 0 || mode < 0 || mode > 1) {
    set_error("stack_batch: bad arguments (W <= T < 2^31, 1 <= P <= W, mode 0 mean, 1 max)");
    return -1;
  }
  const Windows win((int)T, W, P);
  const long long nw = (long long)S * win.K;
  if (w0 >= nw) return 0;
  const int nb = (int)std::min<long long>(B, nw - w0);
  const int s0 = (int)(w0 / win.K), s1 = (int)((w0 + nb - 1) / win.K);
  const long long span = std::min<long long>(T, (long long)(nb - 1) * P + W);
  const dim3 grid((unsigned)((span + ST_NT - 1) / ST_NT), (unsigned)(s1 - s0 + 1), 3);
  stack_batch_kernel<<<grid, ST_NT, 0, (cudaStream_t)stream>>>(y, S, win, w0, nb, s0, mode, probs);
  note_launch();
  return check_launch("stack_batch");
}

int seist_stack_finish(float* probs, int32_t S, int64_t T, int32_t W, int32_t P, void* stream) {
  if (!probs || S <= 0 || W < 1 || T < W || T > INT32_MAX || P < 1 || P > W) {
    set_error("stack_finish: bad arguments (W <= T < 2^31, 1 <= P <= W)");
    return -1;
  }
  const long long n = (long long)S * 3 * T;
  const long long g = std::min<long long>((n + ST_NT - 1) / ST_NT, 132LL * 16);
  stack_finish_kernel<<<(unsigned)g, ST_NT, 0, (cudaStream_t)stream>>>(probs, Windows((int)T, W, P), n);
  note_launch();
  return check_launch("stack_finish");
}

int64_t seist_peaks_work_bytes(int32_t S, int64_t T) {
  if (S <= 0 || T < 3 || T > INT32_MAX) return -1;
  return (int64_t)PeakWork(nullptr, S, (int)T).bytes;
}

int seist_peaks_long(const float* prob, int32_t S, int32_t C, int32_t channel, int64_t T, float mph, int32_t min_peak_dist, void* work,
                     int64_t work_bytes, int64_t* counts, void* stream) {
  if (!prob || !work || !counts || S <= 0 || S > 65535 || T < 3 || T > INT32_MAX || channel < 0 || channel >= C || min_peak_dist <= 1 ||
      work_bytes < seist_peaks_work_bytes(S, T)) {
    set_error("peaks_long: bad arguments (3 <= T < 2^31, S <= 65535, min_peak_dist > 1, work >= seist_peaks_work_bytes)");
    return -1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const PeakWork w(work, S, (int)T);
  const int capc = st_capc((int)T), nblk_t = st_nblk((int)T), nblk_c = st_nblk(capc);
  const float* x = prob + (size_t)channel * T;
  const long long ns = (long long)C * T;
  cand_count_kernel<<<dim3(nblk_t, S), ST_NT, 0, st>>>(x, ns, 1, (int)T - 2, mph, w.blk, nblk_t);
  scan_rows_kernel<<<S, ST_SCAN_NT, 0, st>>>(w.blk, nblk_t, w.ncand, nullptr);
  cand_fill_kernel<<<dim3(nblk_t, S), ST_NT, 0, st>>>(x, ns, 1, (int)T - 2, mph, w.blk, nblk_t, nullptr, 0, capc, w.cidx, w.cval);
  cluster_kernel<<<dim3((capc + CL_SEG - 1) / CL_SEG, S), ST_NT, 0, st>>>(w.ncand, capc, w.cidx, w.cval, w.state, min_peak_dist);
  keep_count_kernel<<<dim3(nblk_c, S), ST_NT, 0, st>>>(w.ncand, capc, w.state, w.blk, nblk_c);
  scan_rows_kernel<<<S, ST_SCAN_NT, 0, st>>>(w.blk, nblk_c, w.nkeep, (long long*)counts);
  for (int i = 0; i < 6; ++i) note_launch();
  return check_launch("peaks_long");
}

int seist_peaks_long_fill(int32_t S, int64_t T, const void* work, int64_t work_bytes, const int64_t* offsets, int64_t* index, float* value,
                          void* stream) {
  if (!work || !offsets || S <= 0 || S > 65535 || T < 3 || T > INT32_MAX || work_bytes < seist_peaks_work_bytes(S, T)) {
    set_error("peaks_long_fill: bad arguments (the work buffer of the seist_peaks_long call)");
    return -1;
  }
  const PeakWork w(const_cast<void*>(work), S, (int)T);
  const int capc = st_capc((int)T), nblk_c = st_nblk(capc);
  keep_fill_kernel<<<dim3(nblk_c, S), ST_NT, 0, (cudaStream_t)stream>>>(w.ncand, capc, w.cidx, w.cval, w.state, w.blk, nblk_c,
                                                                        (const long long*)offsets, 0, (long long*)index, value);
  note_launch();
  return check_launch("peaks_long_fill");
}

int64_t seist_runs_work_bytes(int32_t S, int64_t T) {
  if (S <= 0 || T < 1 || T > INT32_MAX) return -1;
  return (int64_t)run_work_bytes(S, (int)T);
}

int seist_runs_long(const float* prob, int32_t S, int32_t C, int32_t channel, int64_t T, float threshold, void* work, int64_t work_bytes,
                    int64_t* counts, void* stream) {
  if (!prob || !work || !counts || S <= 0 || S > 65535 || T < 1 || T > INT32_MAX || channel < 0 || channel >= C ||
      work_bytes < seist_runs_work_bytes(S, T)) {
    set_error("runs_long: bad arguments (1 <= T < 2^31, S <= 65535, work >= seist_runs_work_bytes)");
    return -1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  int* total = (int*)work;
  int* blk = (int*)((char*)work + st_align(sizeof(int) * S));
  const int nblk = st_nblk((int)T);
  run_count_kernel<<<dim3(nblk, S), ST_NT, 0, st>>>(prob + (size_t)channel * T, (long long)C * T, (int)T, threshold, blk, nblk);
  scan_rows_kernel<<<S, ST_SCAN_NT, 0, st>>>(blk, nblk, total, (long long*)counts);
  note_launch();
  note_launch();
  return check_launch("runs_long");
}

int seist_runs_long_fill(const float* prob, int32_t S, int32_t C, int32_t channel, int64_t T, float threshold, const void* work,
                         int64_t work_bytes, const int64_t* offsets, int64_t* pairs, void* stream) {
  if (!prob || !work || !offsets || S <= 0 || S > 65535 || T < 1 || T > INT32_MAX || channel < 0 || channel >= C ||
      work_bytes < seist_runs_work_bytes(S, T)) {
    set_error("runs_long_fill: bad arguments (the work buffer of the seist_runs_long call)");
    return -1;
  }
  const int* blk = (const int*)((const char*)work + st_align(sizeof(int) * S));
  const int nblk = st_nblk((int)T);
  run_fill_kernel<<<dim3(nblk, S), ST_NT, 0, (cudaStream_t)stream>>>(prob + (size_t)channel * T, (long long)C * T, (int)T, threshold,
                                                                     blk, nblk, (const long long*)offsets, (long long*)pairs);
  note_launch();
  return check_launch("runs_long_fill");
}

uint64_t seist_sizeof_stream_step(void) { return sizeof(SeistStreamStep); }

static bool ss_ok(const SeistStreamStep* p) {
  return p && p->S > 0 && p->S <= 65535 && p->C > 0 && p->W >= 1 && p->W <= 49152 && p->P >= 1 && p->P <= p->W && p->f0 >= 0 &&
         p->r0 >= p->f0 && p->r0 - p->f0 <= p->W && p->r1 >= p->r0 && p->f1 >= p->f0 && p->f1 <= p->r1 && p->r1 - p->f1 <= p->W &&
         p->r1 - p->f0 <= INT32_MAX && p->k0 >= 0 && p->nk >= 0 && p->norm_mode >= 0 && p->norm_mode <= 2 && p->stack_mode >= 0 &&
         p->stack_mode <= 1 && (p->nk == 0 || (p->k0 + p->nk - 1) * p->P + p->W <= p->r1) &&
         (p->tail < 0 || (p->tail >= p->r1 - p->W && p->tail + p->W == p->r1 && p->kr >= 0));
}

int seist_stream_window(const SeistStreamStep* step, const float* tail_raw, const float* chunk, int64_t j0, int32_t B, float* x,
                        void* stream) {
  if (!ss_ok(step) || !x || j0 < 0 || B <= 0 || (step->r0 > 0 && !tail_raw) || (step->r1 > step->r0 && !chunk)) {
    set_error("stream_window: bad arguments (a consistent SeistStreamStep, W <= 49152, j0 >= 0, B > 0)");
    return -1;
  }
  static int attr = 0;
  const int smem = (int)sizeof(float) * step->W;
  if (smem > 48 * 1024 && smem > attr) {
    cudaFuncSetAttribute(stream_window_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr = smem;
  }
  stream_window_kernel<<<(unsigned)((long long)B * step->C), PR_NT, smem, (cudaStream_t)stream>>>(*step, tail_raw, chunk, j0, x);
  note_launch();
  return check_launch("stream_window");
}

int seist_stream_stack(const SeistStreamStep* step, const float* y, int64_t j0, int32_t B, const float* carry, float* acc,
                       void* stream) {
  if (!ss_ok(step) || !y || !carry || !acc || j0 < 0 || B <= 0) {
    set_error("stream_stack: bad arguments (a consistent SeistStreamStep, j0 >= 0, B > 0)");
    return -1;
  }
  const SeistStreamStep& p = *step;
  const long long nw = p.nk + (p.tail >= 0 ? 1 : 0), total = (long long)p.S * nw;
  if (j0 >= total) return 0;
  const int nb = (int)std::min<long long>(B, total - j0);
  const int s0 = (int)(j0 / nw), s1 = (int)((j0 + nb - 1) / nw);
  const long long span = std::min<long long>(p.r1 - p.f0, (long long)(nb - 1) * p.P + p.W);
  const dim3 grid((unsigned)((span + ST_NT - 1) / ST_NT), (unsigned)(s1 - s0 + 1), 3);
  stream_stack_kernel<<<grid, ST_NT, 0, (cudaStream_t)stream>>>(p, y, j0, nb, s0, carry, acc);
  note_launch();
  return check_launch("stream_stack");
}

int seist_stream_emit(const SeistStreamStep* step, const float* carry, const float* acc, float* probs, float* carry_out,
                      void* stream) {
  if (!ss_ok(step) || !carry || !carry_out || (step->r1 > step->f0 && !acc) || (step->f1 > step->f0 && !probs)) {
    set_error("stream_emit: bad arguments (a consistent SeistStreamStep)");
    return -1;
  }
  const long long n = (long long)step->S * 3 * (step->r1 - step->f0);
  if (n == 0) return 0;
  const long long g = std::min<long long>((n + ST_NT - 1) / ST_NT, 132LL * 16);
  stream_emit_kernel<<<(unsigned)g, ST_NT, 0, (cudaStream_t)stream>>>(*step, carry, acc, probs, carry_out);
  note_launch();
  return check_launch("stream_emit");
}

int seist_stream_keep(const SeistStreamStep* step, const float* tail_raw, const float* chunk, float* tail_out, void* stream) {
  if (!ss_ok(step) || !tail_out || (step->r0 > 0 && !tail_raw) || (step->r1 > step->r0 && !chunk) || step->S * step->C > 65535) {
    set_error("stream_keep: bad arguments (a consistent SeistStreamStep, S * C <= 65535)");
    return -1;
  }
  const long long keep = std::min<long long>(step->W, step->r1);
  if (keep == 0) return 0;
  stream_keep_kernel<<<dim3((unsigned)((keep + ST_NT - 1) / ST_NT), step->S * step->C), ST_NT, 0, (cudaStream_t)stream>>>(
      *step, tail_raw, chunk, tail_out);
  note_launch();
  return check_launch("stream_keep");
}

int64_t seist_stream_peaks_work_bytes(int32_t S, int32_t capc, int64_t L) {
  if (S <= 0 || capc < 1 || L < 2 || L > INT32_MAX) return -1;
  return (int64_t)StreamPeakWork(nullptr, S, capc, L).bytes;
}

uint64_t seist_sizeof_ragged_step(void) { return sizeof(SeistRaggedStep); }

static bool rg_ok(const SeistRaggedStep* p) {
  return p && p->f0 && p->r0 && p->f1 && p->r1 && p->k0 && p->nk && p->tail && p->kr && p->win_off && p->chunk_off && p->acc_off &&
         p->out_off && p->S > 0 && p->S <= 65535 && p->C > 0 && p->W >= 1 && p->W <= 49152 && p->P >= 1 && p->P <= p->W &&
         p->n_win >= 0 && p->max_len >= 0 && p->max_len <= INT32_MAX && p->norm_mode >= 0 && p->norm_mode <= 2 &&
         p->stack_mode >= 0 && p->stack_mode <= 1;
}

int seist_ragged_window(const SeistRaggedStep* step, const float* tail_raw, const float* chunk, int64_t j0, int32_t B, float* x,
                        void* stream) {
  if (!rg_ok(step) || !tail_raw || !chunk || !x || j0 < 0 || B <= 0 || (long long)B * step->C > INT32_MAX) {
    set_error("ragged_window: bad arguments (a consistent SeistRaggedStep, W <= 49152, non-null tail_raw and chunk, j0 >= 0, B > 0)");
    return -1;
  }
  static int attr = 0;
  const int smem = (int)sizeof(float) * step->W;
  if (smem > 48 * 1024 && smem > attr) {
    cudaFuncSetAttribute(ragged_window_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr = smem;
  }
  ragged_window_kernel<<<(unsigned)((long long)B * step->C), PR_NT, smem, (cudaStream_t)stream>>>(*step, tail_raw, chunk, j0, x);
  note_launch();
  return check_launch("ragged_window");
}

int seist_ragged_stack(const SeistRaggedStep* step, const float* y, int64_t j0, int32_t B, int32_t s0, int32_t s1,
                       const float* carry, float* acc, void* stream) {
  if (!rg_ok(step) || !y || !carry || !acc || j0 < 0 || B <= 0 || s0 < 0 || s1 < s0 || s1 >= step->S) {
    set_error("ragged_stack: bad arguments (a consistent SeistRaggedStep, j0 >= 0, B > 0, 0 <= s0 <= s1 < S)");
    return -1;
  }
  const SeistRaggedStep& p = *step;
  if (j0 >= p.n_win) return 0;
  const int nb = (int)std::min<long long>(B, p.n_win - j0);
  const long long span = std::min<long long>(p.max_len, (long long)(nb - 1) * p.P + p.W);
  if (span == 0) return 0;
  const dim3 grid((unsigned)((span + ST_NT - 1) / ST_NT), (unsigned)(s1 - s0 + 1), 3);
  ragged_stack_kernel<<<grid, ST_NT, 0, (cudaStream_t)stream>>>(p, y, j0, nb, s0, carry, acc);
  note_launch();
  return check_launch("ragged_stack");
}

int seist_ragged_emit(const SeistRaggedStep* step, const float* carry, const float* acc, float* probs, float* carry_out,
                      void* stream) {
  if (!rg_ok(step) || !carry || !acc || !probs || !carry_out || carry_out == carry) {
    set_error("ragged_emit: bad arguments (a consistent SeistRaggedStep, non-null buffers, carry_out distinct from carry)");
    return -1;
  }
  if (step->max_len == 0) return 0;
  const dim3 grid((unsigned)((step->max_len + ST_NT - 1) / ST_NT), (unsigned)step->S, 3);
  ragged_emit_kernel<<<grid, ST_NT, 0, (cudaStream_t)stream>>>(*step, carry, acc, probs, carry_out);
  note_launch();
  return check_launch("ragged_emit");
}

int seist_ragged_keep(const SeistRaggedStep* step, const float* tail_raw, const float* chunk, float* tail_out, void* stream) {
  if (!rg_ok(step) || !tail_raw || !chunk || !tail_out || tail_out == tail_raw || step->S * step->C > 65535) {
    set_error("ragged_keep: bad arguments (a consistent SeistRaggedStep, S * C <= 65535, tail_out distinct from tail_raw)");
    return -1;
  }
  const dim3 grid((unsigned)((step->W + ST_NT - 1) / ST_NT), (unsigned)(step->S * step->C));
  ragged_keep_kernel<<<grid, ST_NT, 0, (cudaStream_t)stream>>>(*step, tail_raw, chunk, tail_out);
  note_launch();
  return check_launch("ragged_keep");
}

int seist_ragged_history(const float* held, const int64_t* held_off, const int64_t* h0_held, int64_t held_capacity, const float* chunk,
                         const int64_t* chunk_off, int64_t chunk_capacity, const int64_t* h0_out, const int64_t* out_off, int32_t S,
                         int32_t C, int64_t max_len, float* out, int64_t out_capacity, void* stream) {
  if (!held || !held_off || !h0_held || !chunk || !chunk_off || !h0_out || !out_off || !out || out == held || out == chunk || S <= 0 ||
      C <= 0 || (long long)S * C > 65535 || held_capacity < 0 || chunk_capacity < 0 || out_capacity < 0 || max_len < 0 ||
      max_len > INT32_MAX) {
    set_error("ragged_history: bad arguments (non-null buffers and per-station arrays, out distinct from held and chunk, "
              "S * C <= 65535, 0 <= max_len < 2^31, capacities >= 0)");
    return -1;
  }
  if (max_len == 0) return 0;
  const dim3 grid((unsigned)((max_len + ST_NT - 1) / ST_NT), (unsigned)(S * C));
  ragged_history_kernel<<<grid, ST_NT, 0, (cudaStream_t)stream>>>(
      held, (const long long*)held_off, (const long long*)h0_held, held_capacity, chunk, (const long long*)chunk_off, chunk_capacity,
      (const long long*)h0_out, (const long long*)out_off, C, out, out_capacity);
  note_launch();
  return check_launch("ragged_history");
}

int seist_ragged_event_windows(const float* hist, const int64_t* hist_off, const int64_t* h0, int64_t hist_capacity, int32_t S,
                               int32_t C, const int64_t* index, int64_t M, const int64_t* offsets, int64_t e0, int32_t B, int32_t W,
                               int32_t anchor, int32_t mode, float* const* x, int32_t n_dst, void* stream) {
  bool ok = hist && hist_off && h0 && hist_capacity >= 0 && (index || M == 0) && offsets && x && S > 0 && C > 0 && M >= 0 &&
            e0 >= 0 && B > 0 && (long long)B * C <= INT32_MAX && W >= 1 && W <= 49152 && anchor >= 0 && anchor <= W && mode >= 0 &&
            mode <= 2 && n_dst >= 1 && n_dst <= EW_MAX_DST;
  EventDst dst{};
  for (int d = 0; ok && d < n_dst; ++d) ok = (dst.x[d] = x[d]) != nullptr;
  if (!ok) {
    set_error("ragged_event_windows: bad arguments (non-null history and per-station arrays, 1 <= W <= 49152, 0 <= anchor <= W, "
              "M >= 0, e0 >= 0, B > 0, mode 0 none, 1 std, 2 max, 1 to 4 non-null destinations)");
    return -1;
  }
  static int attr = 0;
  const int smem = (int)sizeof(float) * W;
  if (smem > 48 * 1024 && smem > attr) {
    cudaFuncSetAttribute(ragged_event_windows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr = smem;
  }
  ragged_event_windows_kernel<<<(unsigned)((long long)B * C), PR_NT, smem, (cudaStream_t)stream>>>(
      hist, (const long long*)hist_off, (const long long*)h0, hist_capacity, S, C, (const long long*)index, (const long long*)offsets, M,
      e0, W, anchor, mode, dst, n_dst);
  note_launch();
  return check_launch("ragged_event_windows");
}

int seist_gap_event_windows(const float* hist, const int64_t* hist_off, const int64_t* h0, int64_t hist_capacity, int32_t S, int32_t C,
                            const int64_t* pos_station, const int64_t* pos_on, const int64_t* pos_end, const int64_t* pos_off,
                            int32_t n_pos, const int64_t* index, int64_t M, int64_t e0, int32_t B, int32_t W, int32_t anchor, int32_t mode,
                            float* const* x, int32_t n_dst, void* stream) {
  bool ok = hist && hist_off && h0 && hist_capacity >= 0 && pos_station && pos_on && pos_end && pos_off && n_pos >= 1 &&
            (index || M == 0) && x && S > 0 && C > 0 && M >= 0 && e0 >= 0 && B > 0 && (long long)B * C <= INT32_MAX && W >= 1 &&
            W <= 49152 && anchor >= 0 && anchor <= W && mode >= 0 && mode <= 2 && n_dst >= 1 && n_dst <= EW_MAX_DST;
  EventDst dst{};
  for (int d = 0; ok && d < n_dst; ++d) ok = (dst.x[d] = x[d]) != nullptr;
  if (!ok) {
    set_error("gap_event_windows: bad arguments (non-null history, per-station arrays and position table, n_pos >= 1, "
              "1 <= W <= 49152, 0 <= anchor <= W, M >= 0, e0 >= 0, B > 0, mode 0 none, 1 std, 2 max, 1 to 4 non-null destinations)");
    return -1;
  }
  static int attr = 0;
  const int smem = (int)sizeof(float) * W;
  if (smem > 48 * 1024 && smem > attr) {
    cudaFuncSetAttribute(gap_event_windows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr = smem;
  }
  gap_event_windows_kernel<<<(unsigned)((long long)B * C), PR_NT, smem, (cudaStream_t)stream>>>(
      hist, (const long long*)hist_off, (const long long*)h0, hist_capacity, S, C, (const long long*)pos_station, (const long long*)pos_on,
      (const long long*)pos_end, (const long long*)pos_off, n_pos, (const long long*)index, M, e0, W, anchor, mode, dst, n_dst);
  note_launch();
  return check_launch("gap_event_windows");
}

int seist_ragged_ext(const float* look, const float* probs, const int64_t* prob_off, const int64_t* ext_off, int32_t S, int32_t C,
                     int64_t max_L, float* ext, float* look_out, void* stream) {
  if (!look || !probs || !prob_off || !ext_off || !ext || !look_out || look_out == look || S <= 0 || S > 65535 || C <= 0 ||
      C > 65535 || max_L < 2 || max_L > INT32_MAX) {
    set_error("ragged_ext: bad arguments (non-null buffers, look_out distinct from look, S, C <= 65535, 2 <= max_L < 2^31)");
    return -1;
  }
  const dim3 grid((unsigned)((max_L + ST_NT - 1) / ST_NT), (unsigned)S, (unsigned)C);
  ragged_ext_kernel<<<grid, ST_NT, 0, (cudaStream_t)stream>>>(look, probs, (const long long*)prob_off, (const long long*)ext_off, C, ext,
                                                              look_out);
  note_launch();
  return check_launch("ragged_ext");
}

static bool rg_rows_ok(const float* ext, const int64_t* ext_off, int32_t S, int32_t C, int32_t channel, int64_t max_L, const int64_t* lo,
                       const int64_t* hi, int64_t max_span) {
  return ext && ext_off && lo && hi && S > 0 && S <= 65535 && channel >= 0 && channel < C && max_L >= 2 && max_L <= INT32_MAX &&
         max_span >= 0 && max_span <= max_L;
}

int seist_ragged_peaks(const float* ext, const int64_t* ext_off, int32_t S, int32_t C, int32_t channel, int64_t max_L,
                       const int64_t* lo, const int64_t* hi, int64_t max_span, float mph, int32_t min_peak_dist,
                       const int64_t* lim, const int64_t* base, const int64_t* ishift, void* work, int32_t capc,
                       const void* prev, int32_t prev_capc, int64_t prev_L, const int64_t* delta, int32_t max_pend,
                       int64_t* counts, int64_t* info, void* stream) {
  if (!rg_rows_ok(ext, ext_off, S, C, channel, max_L, lo, hi, max_span) || !lim || !base || !ishift || !work || !counts || !info ||
      min_peak_dist <= 1 || max_pend < 0 || (long long)capc < (long long)max_pend + max_L / 2 + 1 ||
      (prev && (!delta || prev_capc < 1 || prev_L < 2 || prev_L > INT32_MAX))) {
    set_error("ragged_peaks: bad arguments (2 <= max_L < 2^31, 0 <= max_span <= max_L, S <= 65535, min_peak_dist > 1, "
              "capc >= max_pend + max_L / 2 + 1, per-row arrays non-null)");
    return -1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const StreamPeakWork w(work, S, capc, max_L);
  const int nb = std::max(1, st_nblk((int)max_span)), nbc = st_nblk(capc);
  const StreamPeakWork pw(prev, S, prev ? prev_capc : 1, prev ? prev_L : 2);
  const long long* eo = (const long long*)ext_off;
  const long long *lo_a = (const long long*)lo, *hi_a = (const long long*)hi;
  rg_pend_move_kernel<<<dim3(std::max(1, (max_pend + ST_NT - 1) / ST_NT), S), ST_NT, 0, st>>>(
      prev ? pw.cidx : nullptr, pw.cval, prev_capc, pw.nclosed, pw.ncand, (const long long*)delta, w.cidx, w.cval, capc, w.npend);
  rg_cand_count_kernel<<<dim3(nb, S), ST_NT, 0, st>>>(ext, eo, C, channel, lo_a, hi_a, mph, w.blk, nb);
  scan_rows_kernel<<<S, ST_SCAN_NT, 0, st>>>(w.blk, nb, w.nnew, nullptr);
  rg_cand_fill_kernel<<<dim3(nb, S), ST_NT, 0, st>>>(ext, eo, C, channel, lo_a, hi_a, mph, w.blk, nb, w.npend,
                                                     (const long long*)ishift, capc, w.cidx, w.cval);
  rg_close_scan_kernel<<<S, ST_NT, 0, st>>>(w.npend, w.nnew, w.cidx, capc, min_peak_dist, (const long long*)lim, (const long long*)base,
                                            w.ncand, w.nclosed, (long long*)info);
  cluster_kernel<<<dim3((capc + CL_SEG - 1) / CL_SEG, S), ST_NT, 0, st>>>(w.nclosed, capc, w.cidx, w.cval, w.state, min_peak_dist);
  keep_count_kernel<<<dim3(nbc, S), ST_NT, 0, st>>>(w.nclosed, capc, w.state, w.blk, nbc);
  scan_rows_kernel<<<S, ST_SCAN_NT, 0, st>>>(w.blk, nbc, w.nkeep, (long long*)counts);
  for (int i = 0; i < 8; ++i) note_launch();
  return check_launch("ragged_peaks");
}

int seist_ragged_peaks_fill(int32_t S, int64_t max_L, const void* work, int32_t capc, const int64_t* base, const int64_t* offsets,
                            int64_t* index, float* value, void* stream) {
  if (!work || !base || !offsets || !index || !value || S <= 0 || S > 65535 || max_L < 2 || max_L > INT32_MAX || capc < 1) {
    set_error("ragged_peaks_fill: bad arguments (the work buffer of the seist_ragged_peaks call, non-null outputs)");
    return -1;
  }
  const StreamPeakWork w(const_cast<void*>(work), S, capc, max_L);
  const int nbc = st_nblk(capc);
  rg_keep_fill_kernel<<<dim3(nbc, S), ST_NT, 0, (cudaStream_t)stream>>>(w.nclosed, capc, w.cidx, w.cval, w.state, w.blk, nbc,
                                                                        (const long long*)offsets, (const long long*)base,
                                                                        (long long*)index, value);
  note_launch();
  return check_launch("ragged_peaks_fill");
}

int seist_ragged_runs(const float* ext, const int64_t* ext_off, int32_t S, int32_t C, int32_t channel, int64_t max_L,
                      const int64_t* lo, const int64_t* hi, int64_t max_span, float threshold, const int64_t* open_in,
                      int64_t* open_out, void* work, int64_t work_bytes, int64_t* counts, void* stream) {
  if (!rg_rows_ok(ext, ext_off, S, C, channel, max_L, lo, hi, max_span) || !open_in || !open_out || !work || !counts ||
      work_bytes < seist_runs_work_bytes(S, max_L)) {
    set_error("ragged_runs: bad arguments (2 <= max_L < 2^31, 0 <= max_span <= max_L, S <= 65535, "
              "work >= seist_runs_work_bytes(S, max_L))");
    return -1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  int* total = (int*)work;
  int* blk = (int*)((char*)work + st_align(sizeof(int) * S));
  const int nb = std::max(1, st_nblk((int)max_span));
  rg_srun_count_kernel<<<dim3(nb, S), ST_NT, 0, st>>>(ext, (const long long*)ext_off, C, channel, (const long long*)lo,
                                                      (const long long*)hi, threshold, blk, nb, (const long long*)open_in,
                                                      (long long*)open_out);
  scan_rows_kernel<<<S, ST_SCAN_NT, 0, st>>>(blk, nb, total, (long long*)counts);
  note_launch();
  note_launch();
  return check_launch("ragged_runs");
}

int seist_ragged_runs_fill(const float* ext, const int64_t* ext_off, int32_t S, int32_t C, int32_t channel, int64_t max_L,
                           const int64_t* lo, const int64_t* hi, int64_t max_span, float threshold, const int64_t* g0,
                           const int64_t* open_in, int64_t* open_out, const void* work, int64_t work_bytes,
                           const int64_t* offsets, int64_t* pairs, void* stream) {
  if (!rg_rows_ok(ext, ext_off, S, C, channel, max_L, lo, hi, max_span) || !g0 || !open_in || !open_out || !work || !offsets ||
      work_bytes < seist_runs_work_bytes(S, max_L)) {
    set_error("ragged_runs_fill: bad arguments (the work buffer of the seist_ragged_runs call, per-row arrays non-null)");
    return -1;
  }
  const int* blk = (const int*)((const char*)work + st_align(sizeof(int) * S));
  const int nb = std::max(1, st_nblk((int)max_span));
  rg_srun_fill_kernel<<<dim3(nb, S), ST_NT, 0, (cudaStream_t)stream>>>(ext, (const long long*)ext_off, C, channel, (const long long*)lo,
                                                                       (const long long*)hi, threshold, (const long long*)g0, blk, nb,
                                                                       (const long long*)offsets, (const long long*)open_in,
                                                                       (long long*)open_out, (long long*)pairs);
  note_launch();
  return check_launch("ragged_runs_fill");
}

int seist_gap_segments(const float* record, int32_t S, int32_t C, int64_t T, void* work, int64_t work_bytes, int64_t* counts,
                       void* stream) {
  if (!record || !work || !counts || S <= 0 || S > 65535 || C <= 0 || T < 1 || T > INT32_MAX || work_bytes < seist_runs_work_bytes(S, T)) {
    set_error("gap_segments: bad arguments (1 <= T < 2^31, 1 <= S <= 65535, C >= 1, work >= seist_runs_work_bytes(S, T))");
    return -1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  int* total = (int*)work;
  int* blk = (int*)((char*)work + st_align(sizeof(int) * S));
  const int nblk = st_nblk((int)T);
  gap_count_kernel<<<dim3(nblk, S), ST_NT, 0, st>>>(record, C, (int)T, blk, nblk);
  scan_rows_kernel<<<S, ST_SCAN_NT, 0, st>>>(blk, nblk, total, (long long*)counts);
  note_launch();
  note_launch();
  return check_launch("gap_segments");
}

int seist_gap_segments_fill(const float* record, int32_t S, int32_t C, int64_t T, const void* work, int64_t work_bytes,
                            const int64_t* offsets, int64_t* pairs, int64_t capacity, void* stream) {
  if (!record || !work || !offsets || !pairs || S <= 0 || S > 65535 || C <= 0 || T < 1 || T > INT32_MAX || capacity < 0 ||
      work_bytes < seist_runs_work_bytes(S, T)) {
    set_error("gap_segments_fill: bad arguments (the work buffer of the seist_gap_segments call, non-null pairs, capacity >= 0)");
    return -1;
  }
  const int* blk = (const int*)((const char*)work + st_align(sizeof(int) * S));
  const int nblk = st_nblk((int)T);
  gap_fill_kernel<<<dim3(nblk, S), ST_NT, 0, (cudaStream_t)stream>>>(record, C, (int)T, blk, nblk, (const long long*)offsets, capacity,
                                                                     (long long*)pairs);
  note_launch();
  return check_launch("gap_segments_fill");
}

static bool sg_ok(int32_t S, int64_t T, const int64_t* pairs, const int64_t* per_seg, int32_t G, int32_t W, int32_t P) {
  return pairs && per_seg && S > 0 && S <= 65535 && T >= 1 && T <= INT32_MAX && G >= 1 && W >= 1 && W <= 49152 && P >= 1 && P <= W;
}

int seist_segment_window(const float* record, int32_t S, int32_t C, int64_t T, const int64_t* pairs, const int64_t* station,
                         const int64_t* win_off, int32_t G, int64_t n_win, int32_t W, int32_t P, int64_t j0, int32_t B, int32_t mode,
                         float* x, void* stream) {
  if (!sg_ok(S, T, pairs, station, G, W, P) || !record || !win_off || !x || C <= 0 || n_win < 0 || j0 < 0 || B <= 0 ||
      (long long)B * C > INT32_MAX || mode < 0 || mode > 2) {
    set_error("segment_window: bad arguments (1 <= T < 2^31, 1 <= S <= 65535, G >= 1, 1 <= P <= W <= 49152, n_win >= 0, j0 >= 0, "
              "B > 0, mode 0 none, 1 std, 2 max)");
    return -1;
  }
  static int attr = 0;
  const int smem = (int)sizeof(float) * W;
  if (smem > 48 * 1024 && smem > attr) {
    cudaFuncSetAttribute(segment_window_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr = smem;
  }
  segment_window_kernel<<<(unsigned)((long long)B * C), PR_NT, smem, (cudaStream_t)stream>>>(
      record, S, C, T, (const long long*)pairs, (const long long*)station, (const long long*)win_off, G, n_win, W, P, j0, mode, x);
  note_launch();
  return check_launch("segment_window");
}

int seist_segment_stack(const float* y, int32_t S, int64_t T, const int64_t* pairs, const int64_t* station, const int64_t* win_off,
                        int32_t G, int64_t n_win, int32_t W, int32_t P, int64_t j0, int32_t B, int32_t g0, int32_t g1, int32_t mode,
                        float* probs, void* stream) {
  if (!sg_ok(S, T, pairs, station, G, W, P) || !y || !win_off || !probs || n_win < 0 || j0 < 0 || B <= 0 || g0 < 0 || g1 < g0 ||
      g1 >= G || mode < 0 || mode > 1) {
    set_error("segment_stack: bad arguments (1 <= T < 2^31, 1 <= S <= 65535, 1 <= P <= W <= 49152, j0 >= 0, B > 0, "
              "0 <= g0 <= g1 < G, mode 0 mean, 1 max)");
    return -1;
  }
  if (j0 >= n_win) return 0;
  const int nb = (int)std::min<long long>(B, n_win - j0);
  const long long span = std::min<long long>(T, (long long)(nb - 1) * P + W);
  // short segments between two annotated ones hold no windows but are rows of the grid: more than 65535 of them in one
  // batch take more than one launch
  for (int gs = g0; gs <= g1; gs += 65535) {
    const dim3 grid((unsigned)((span + ST_NT - 1) / ST_NT), (unsigned)std::min(65535, g1 - gs + 1), 3);
    segment_stack_kernel<<<grid, ST_NT, 0, (cudaStream_t)stream>>>(y, S, T, (const long long*)pairs, (const long long*)station,
                                                                   (const long long*)win_off, G, W, P, j0, nb, gs, mode, probs);
    note_launch();
    if (g1 - gs < 65535) break;
  }
  return check_launch("segment_stack");
}

int seist_segment_finish(float* probs, int32_t S, int64_t T, const int64_t* pairs, const int64_t* seg_off, int32_t G, int32_t W,
                         int32_t P, int32_t mode, void* stream) {
  if (!probs || !seg_off || S <= 0 || S > 65535 || T < 1 || T > INT32_MAX || G < 0 || (G > 0 && !pairs) || W < 1 || W > 49152 || P < 1 ||
      P > W || mode < 0 || mode > 1) {
    set_error("segment_finish: bad arguments (1 <= T < 2^31, 1 <= S <= 65535, G >= 0, 1 <= P <= W <= 49152, mode 0 mean, 1 max)");
    return -1;
  }
  const long long n = (long long)S * 3 * T;
  const long long g = std::min<long long>((n + ST_NT - 1) / ST_NT, 132LL * 16);
  segment_finish_kernel<<<(unsigned)g, ST_NT, 0, (cudaStream_t)stream>>>(probs, S, T, (const long long*)pairs, (const long long*)seg_off,
                                                                          G, W, P, mode, n);
  note_launch();
  return check_launch("segment_finish");
}

int seist_segment_gather(const float* probs, int32_t S, int64_t T, const int64_t* pairs, const int64_t* station, int32_t G,
                         const int64_t* rows, const int64_t* prob_off, int32_t n_rows, int64_t max_len, float* flat, int64_t capacity,
                         void* stream) {
  if (!probs || !pairs || !station || !rows || !prob_off || !flat || S <= 0 || S > 65535 || T < 1 || T > INT32_MAX || G < 1 ||
      n_rows < 1 || n_rows > 65535 || max_len < 0 || max_len > INT32_MAX || capacity < 0) {
    set_error("segment_gather: bad arguments (1 <= T < 2^31, 1 <= S <= 65535, G >= 1, 1 <= n_rows <= 65535, 0 <= max_len < 2^31)");
    return -1;
  }
  if (max_len == 0) return 0;
  const dim3 grid((unsigned)((max_len + ST_NT - 1) / ST_NT), (unsigned)n_rows, 3);
  segment_gather_kernel<<<grid, ST_NT, 0, (cudaStream_t)stream>>>(probs, S, T, (const long long*)pairs, (const long long*)station, G,
                                                                  (const long long*)rows, (const long long*)prob_off, capacity, flat);
  note_launch();
  return check_launch("segment_gather");
}

int seist_segment_event_windows(const float* record, int32_t S, int32_t C, int64_t T, const int64_t* pairs, const int64_t* seg_off,
                                const uint8_t* annotated, int32_t G, const int64_t* index, int64_t M, const int64_t* offsets, int64_t e0,
                                int32_t B, int32_t W, int32_t anchor, int32_t mode, float* const* x, int32_t n_dst, void* stream) {
  bool ok = record && seg_off && (G == 0 || (pairs && annotated)) && G >= 0 && (index || M == 0) && offsets && x && S > 0 &&
            S <= 65535 && C > 0 && T >= 1 && T <= INT32_MAX && M >= 0 && e0 >= 0 && B > 0 && (long long)B * C <= INT32_MAX && W >= 1 &&
            W <= 49152 && anchor >= 0 && anchor <= W && mode >= 0 && mode <= 2 && n_dst >= 1 && n_dst <= EW_MAX_DST;
  EventDst dst{};
  for (int d = 0; ok && d < n_dst; ++d) ok = (dst.x[d] = x[d]) != nullptr;
  if (!ok) {
    set_error("segment_event_windows: bad arguments (1 <= T < 2^31, 1 <= S <= 65535, G >= 0, 1 <= W <= 49152, 0 <= anchor <= W, "
              "M >= 0, e0 >= 0, B > 0, mode 0 none, 1 std, 2 max, 1 to 4 non-null destinations)");
    return -1;
  }
  static int attr = 0;
  const int smem = (int)sizeof(float) * W;
  if (smem > 48 * 1024 && smem > attr) {
    cudaFuncSetAttribute(segment_event_windows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr = smem;
  }
  segment_event_windows_kernel<<<(unsigned)((long long)B * C), PR_NT, smem, (cudaStream_t)stream>>>(
      record, S, C, T, (const long long*)pairs, (const long long*)seg_off, annotated, G, (const long long*)index, (const long long*)offsets,
      M, e0, W, anchor, mode, dst, n_dst);
  note_launch();
  return check_launch("segment_event_windows");
}

int seist_gap_stream_scan(const float* chunk, int64_t chunk_capacity, const int64_t* chunk_off, int32_t S, int32_t C, int64_t max_n,
                          void* work, int64_t work_bytes, int64_t* counts, void* stream) {
  if (!chunk || !chunk_off || !work || !counts || S <= 0 || S > 65535 || C <= 0 || max_n < 1 || max_n > INT32_MAX ||
      chunk_capacity < 0 || work_bytes < seist_runs_work_bytes(S, max_n)) {
    set_error("gap_stream_scan: bad arguments (1 <= S <= 65535, C >= 1, 1 <= max_n < 2^31, work >= seist_runs_work_bytes(S, max_n))");
    return -1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  int* total = (int*)work;
  int* blk = (int*)((char*)work + st_align(sizeof(int) * S));
  const int nblk = st_nblk((int)max_n);
  gap_stream_count_kernel<<<dim3(nblk, S), ST_NT, 0, st>>>(chunk, chunk_capacity, (const long long*)chunk_off, C, blk, nblk);
  scan_rows_kernel<<<S, ST_SCAN_NT, 0, st>>>(blk, nblk, total, (long long*)counts);
  note_launch();
  note_launch();
  return check_launch("gap_stream_scan");
}

int seist_gap_stream_fill(const float* chunk, int64_t chunk_capacity, const int64_t* chunk_off, int32_t S, int32_t C, int64_t max_n,
                          const void* work, int64_t work_bytes, const int64_t* offsets, int64_t* pairs, int64_t capacity, void* stream) {
  if (!chunk || !chunk_off || !work || !offsets || !pairs || S <= 0 || S > 65535 || C <= 0 || max_n < 1 || max_n > INT32_MAX ||
      chunk_capacity < 0 || capacity < 0 || work_bytes < seist_runs_work_bytes(S, max_n)) {
    set_error("gap_stream_fill: bad arguments (the work buffer of the seist_gap_stream_scan call, non-null pairs, capacity >= 0)");
    return -1;
  }
  const int* blk = (const int*)((const char*)work + st_align(sizeof(int) * S));
  const int nblk = st_nblk((int)max_n);
  gap_stream_fill_kernel<<<dim3(nblk, S), ST_NT, 0, (cudaStream_t)stream>>>(chunk, chunk_capacity, (const long long*)chunk_off, C, blk,
                                                                            nblk, (const long long*)offsets, capacity, (long long*)pairs);
  note_launch();
  return check_launch("gap_stream_fill");
}

static unsigned gs_grid(long long n) { return (unsigned)std::max<long long>(1, std::min<long long>((n + ST_NT - 1) / ST_NT, 132LL * 16)); }

int seist_gap_stream_pack(const float* chunk, int64_t chunk_capacity, const int64_t* chunk_off, int32_t S, int32_t C,
                          const int64_t* row_station, const int64_t* row_start, const int64_t* row_off, int32_t n_rows, int64_t n,
                          float* out, int64_t out_capacity, void* stream) {
  if (!chunk || !chunk_off || !row_station || !row_start || !row_off || !out || S <= 0 || C <= 0 || n_rows < 1 || n < 0 ||
      chunk_capacity < 0 || out_capacity < 0) {
    set_error("gap_stream_pack: bad arguments (non-null buffers and tables, S, C, n_rows >= 1, n >= 0, capacities >= 0)");
    return -1;
  }
  if (n == 0) return 0;
  gap_stream_pack_kernel<<<gs_grid(n), ST_NT, 0, (cudaStream_t)stream>>>(chunk, chunk_capacity, (const long long*)chunk_off, S, C,
                                                                         (const long long*)row_station, (const long long*)row_start,
                                                                         (const long long*)row_off, n_rows, n, out, out_capacity);
  note_launch();
  return check_launch("gap_stream_pack");
}

int seist_gap_stream_copy(const float* src, int64_t src_capacity, const int64_t* m_off, const int64_t* src_base, const int64_t* src_ld,
                          const int64_t* dst_base, const int64_t* dst_ld, int32_t n_rows, int64_t n, float* dst, int64_t dst_capacity,
                          void* stream) {
  if (!src || !m_off || !src_base || !src_ld || !dst_base || !dst_ld || !dst || src == dst || n_rows < 1 || n < 0 || src_capacity < 0 ||
      dst_capacity < 0) {
    set_error("gap_stream_copy: bad arguments (non-null, distinct buffers and tables, n_rows >= 1, n >= 0, capacities >= 0)");
    return -1;
  }
  if (n == 0) return 0;
  gap_stream_copy_kernel<<<gs_grid(n), ST_NT, 0, (cudaStream_t)stream>>>(src, src_capacity, (const long long*)m_off,
                                                                         (const long long*)src_base, (const long long*)src_ld,
                                                                         (const long long*)dst_base, (const long long*)dst_ld, n_rows, n,
                                                                         dst, dst_capacity);
  note_launch();
  return check_launch("gap_stream_copy");
}

}  // extern "C"
