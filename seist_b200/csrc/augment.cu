// Training-time input pipeline on the device: the reference's `DataPreprocessor.process` (training/preprocess.py:501-542)
// for a whole batch - `_is_noise`, `_pad_phases`, `_data_augmentation` (:432-499), `_cut_window` (:172-222), `_normalize`.
//
// Two kernels.  aug_draw_kernel (one thread per trace) replays the reference's decision sequence on the trace's phase
// list with counter-based uniforms and writes a per-trace recipe plus the output phase lists.  aug_apply_kernel (one CTA
// per trace) stages the raw trace in shared memory, applies the recipe in the reference's order, then cuts and normalises.
// The draws are mirrored bit for bit by tests/augment_ref.py::CounterDraws; every double expression that the oracle
// evaluates as separate Python operations is written with _rn intrinsics so that nvcc cannot contract it into an FMA.
#include "common.cuh"

namespace seist {

constexpr int AUG_NT = 512;                       // apply kernel threads
constexpr int AUG_DRAW_NT = 128;
constexpr int AUG_MAXK = 8;                       // phase list entries (dpk_labels takes K <= 8)
constexpr int AUG_MAXC = 8;
constexpr int AUG_MAXWIN = 1024;                  // mask / noise windows per trace (bitmask of 32 words)
constexpr long long AUG_ABSENT = -1000000;        // entries at or below are "no phase" (Python pads with -10^7)
constexpr uint32_t AUG_STREAM_DRAW = 0x41554700u;
constexpr uint32_t AUG_STREAM_NORMAL = 0x41554710u;   // + 0 generate-noise, 1 add-noise, 2 noise windows

enum : int {
  AUG_F_AUGMENT = 1, AUG_F_DROP = 4, AUG_F_SCALE_MUL = 8, AUG_F_SCALE_DIV = 16, AUG_F_PRE = 32,
  AUG_F_NOISE = 64, AUG_F_GAP = 128, AUG_F_MASKW = 256, AUG_F_NOISEW = 512, AUG_F_NORM64 = 1024,
};

struct AugRecipe {
  int flags, shift, drop_mask, gap_lo, gap_hi, cut, n_fill, n_add;
  float scale;
  int snr[AUG_MAXC];
  int fill_lo[AUG_MAXK], fill_hi[AUG_MAXK];
  int add_src[AUG_MAXK], add_dst[AUG_MAXK], add_len[AUG_MAXK];
  float add_scale[AUG_MAXK];
  uint32_t mask_bits[AUG_MAXWIN / 32], noise_bits[AUG_MAXWIN / 32];
};

// ---- draws -----------------------------------------------------------------------------------------------------------
struct AugRng {
  uint64_t seed, base;
  uint32_t k;
  __device__ double u() { return (double)(rng_u64(seed, AUG_STREAM_DRAW, base + k++) >> 11) * 0x1p-53; }
  __device__ long long randint(long long a, long long b) {   // a + floor(u (b - a)); a when the range is empty
    const double v = u();
    return b > a ? a + (long long)floor(__dmul_rn(v, (double)(b - a))) : a;
  }
  __device__ double uniform(double a, double b) { return __dadd_rn(a, __dmul_rn(u(), b - a)); }
};

// standard normal at counter q of `stream`: Box-Muller on one hash, u1 = (hi + 1) / 2^32 in (0, 1], u2 = lo / 2^32
__device__ __forceinline__ double aug_normal(uint64_t seed, uint32_t stream, uint64_t q) {
  const uint64_t h = rng_u64(seed, stream, q);
  const double u1 = (double)((h >> 32) + 1ull) * 0x1p-32, u2 = (double)(h & 0xFFFFFFFFull) * 0x1p-32;
  return __dmul_rn(sqrt(__dmul_rn(-2.0, log(u1))), cospi(__dmul_rn(2.0, u2)));   // cos(2 pi u2)
}
__device__ __forceinline__ uint64_t aug_nidx(long long n, int C, int c, int i) {
  return (((uint64_t)n * (uint64_t)C + (uint64_t)c) << 16) + (uint64_t)i;
}

__device__ void aug_sort(long long* v, int n) {
  for (int i = 1; i < n; ++i) {
    const long long x = v[i];
    int j = i - 1;
    while (j >= 0 && v[j] > x) { v[j + 1] = v[j]; --j; }
    v[j + 1] = x;
  }
}
// int(spk + coda_ratio * (spk - ppk)): Python float arithmetic, truncation
__device__ __forceinline__ long long aug_coda_end(long long ppk, long long spk, double coda) {
  return (long long)__dadd_rn((double)spk, __dmul_rn(coda, (double)(spk - ppk)));
}
// selection sampling of k of n windows into a bitmask
__device__ void aug_windows(AugRng& r, int n, int k, uint32_t* bits) {
  for (int w = 0; w < AUG_MAXWIN / 32; ++w) bits[w] = 0u;
  int need = k;
  for (int i = 0; i < n && need > 0; ++i)
    if (__dmul_rn((double)(n - i), r.u()) < (double)need) { bits[i >> 5] |= 1u << (i & 31); --need; }
}

__global__ void __launch_bounds__(AUG_DRAW_NT) aug_draw_kernel(
    const long long* __restrict__ ppks_in, const long long* __restrict__ spks_in, int K, const double* __restrict__ snr, int S,
    const uint8_t* __restrict__ augment, long long N, int C, int Lin, SeistAugCfg cfg, const uint64_t* __restrict__ seed_p,
    AugRecipe* __restrict__ rec_out, long long* __restrict__ ppks_out, long long* __restrict__ spks_out, int K_out,
    uint8_t* __restrict__ cleared) {
  const long long n = (long long)blockIdx.x * AUG_DRAW_NT + threadIdx.x;
  if (n >= N) return;
  AugRecipe rec;
  rec.flags = 0; rec.shift = 0; rec.drop_mask = 0; rec.gap_lo = rec.gap_hi = 0; rec.cut = 0; rec.n_fill = 0; rec.n_add = 0;
  rec.scale = 1.f;
  long long p[AUG_MAXK], s[AUG_MAXK];
  int np = 0, ns = 0;
  for (int i = 0; i < K; ++i) {
    const long long a = ppks_in[n * K + i], b = spks_in[n * K + i];
    if (a > AUG_ABSENT) p[np++] = a;
    if (b > AUG_ABSENT) s[ns++] = b;
  }
  // _is_noise (:154-170) on the lists in the order given; more P than S picks (the reference raises) count as noise
  bool noise = np != ns || np < 1;
  for (int i = 0; i < np; ++i) noise = noise || p[i] < 0 || p[i] >= Lin;
  for (int i = 0; i < ns; ++i) noise = noise || s[i] < 0 || s[i] >= Lin;
  if (S > 0) {
    bool all_below = true;
    for (int i = 0; i < S; ++i) all_below = all_below && snr[n * S + i] < cfg.min_snr;
    noise = noise || all_below;
  }
  for (int i = 0; i < np && i < ns; ++i) noise = noise || p[i] >= s[i];
  if (noise) np = ns = 0;
  // _pad_phases (:523-525) pads nothing here: a list that passed _is_noise pairs every sorted P before its sorted S
  aug_sort(p, np);
  aug_sort(s, ns);
  AugRng r{load_seed(seed_p), (uint64_t)n << 32, 0u};
  const int gap = cfg.min_event_gap;
  if (!augment || augment[n]) {
    rec.flags |= AUG_F_AUGMENT;
    auto drop_scale = [&]() {                                    // the drop / scale draws shared by both branches
      if (r.u() < cfg.drop_channel_rate) {                       // _drop_channel (:307-321) + _adjust_amplitude
        rec.flags |= AUG_F_DROP;
        if (C >= 2) {
          const int num = (int)r.randint(1, C);
          int cand[AUG_MAXC], nc = C;
          for (int c = 0; c < C; ++c) cand[c] = c;
          for (int d = 0; d < num; ++d) {
            const int j = (int)r.randint(0, nc);
            rec.drop_mask |= 1 << cand[j];
            for (int q = j; q + 1 < nc; ++q) cand[q] = cand[q + 1];
            --nc;
          }
        }
      }
      if (r.u() < cfg.scale_amplitude_rate) {                    // _scale_amplitude (:335-344)
        const bool mul = r.uniform(0.0, 1.0) < 0.5;
        rec.scale = (float)r.uniform(1.0, 3.0);
        rec.flags |= mul ? AUG_F_SCALE_MUL : AUG_F_SCALE_DIV;
      }
    };
    if (r.u() < cfg.generate_noise_rate) {                       // _generate_noise_data (:244-263), the event is cleared
      for (int i = 0; i < np; ++i) {
        long long ce = aug_coda_end(p[i], s[i], cfg.coda_ratio);
        ce = ce < 0 ? 0 : (ce > Lin ? Lin : ce);
        if (p[i] < ce) { rec.fill_lo[rec.n_fill] = (int)p[i]; rec.fill_hi[rec.n_fill] = (int)ce; ++rec.n_fill; }
      }
      np = ns = 0;
      noise = true;
      drop_scale();
    } else {
      const int adds = cfg.max_event_num - np;
      for (int it = 0; it < adds; ++it) {                        // _add_event (:265-292)
        if (r.u() < cfg.add_event_rate && np > 0) {
          const int t = (int)r.randint(0, np);
          const long long ppk = p[t], spk = s[t], ce = aug_coda_end(ppk, spk, cfg.coda_ratio);
          const long long left = ce + gap, right = Lin - (spk - ppk) - gap;
          if (left < right) {
            const long long add = r.randint(left, right);
            const long long space = (Lin - add) < (ce - ppk) ? (Lin - add) : (ce - ppk);
            const double sc = r.u();
            rec.add_src[rec.n_add] = (int)ppk; rec.add_dst[rec.n_add] = (int)add; rec.add_len[rec.n_add] = (int)space;
            rec.add_scale[rec.n_add] = (float)sc; ++rec.n_add;
            p[np++] = add;
            s[ns++] = add + spk - ppk;
            aug_sort(p, np);
            aug_sort(s, ns);
          }
        }
      }
      if (r.u() < cfg.shift_event_rate) {                       // _shift_event (:294-305)
        const long long sh = r.randint(0, Lin);
        rec.shift = (int)sh;
        for (int i = 0; i < np; ++i) p[i] = (p[i] + sh) % Lin;
        for (int i = 0; i < ns; ++i) s[i] = (s[i] + sh) % Lin;
        aug_sort(p, np);
        aug_sort(s, ns);
      }
      drop_scale();
      if (r.u() < cfg.pre_emphasis_rate) rec.flags |= AUG_F_PRE;
      if (r.u() < cfg.add_noise_rate) {                          // _add_noise (:355-368)
        rec.flags |= AUG_F_NOISE;
        for (int c = 0; c < C; ++c) rec.snr[c] = (int)r.randint(10, 50);
      }
      if (r.u() < cfg.add_gap_rate) {                            // _add_gaps (:370-390)
        rec.flags |= AUG_F_GAP;
        long long ph[2 * AUG_MAXK + 1];
        int nph = 0;
        for (int i = 0; i < np; ++i) ph[nph++] = p[i];
        for (int i = 0; i < ns; ++i) ph[nph++] = s[i];
        long long sgt, egt;
        if (nph > 0) {
          ph[nph++] = Lin - 1;
          aug_sort(ph, nph);
          int m = 1;
          for (int i = 1; i < nph; ++i) if (ph[i] != ph[m - 1]) ph[m++] = ph[i];
          const int ip = (int)r.randint(0, m - 1);
          sgt = r.randint(ph[ip], ph[ip + 1]);
          egt = r.randint(sgt, ph[ip + 1]);
        } else {
          sgt = r.randint(0, Lin - 1);
          egt = r.randint(sgt + 1, Lin);
        }
        rec.gap_lo = (int)sgt; rec.gap_hi = (int)egt;
      }
    }
    const int nw = Lin / cfg.window;                             // _add_mask_windows / _add_noise_windows (:392-430)
    if (cfg.mask_percent > 0) { rec.flags |= AUG_F_MASKW; aug_windows(r, nw, nw * min(cfg.mask_percent, 100) / 100, rec.mask_bits); }
    if (cfg.noise_percent > 0) { rec.flags |= AUG_F_NOISEW; aug_windows(r, nw, nw * min(cfg.noise_percent, 100) / 100, rec.noise_bits); }
  }
  // _cut_window (:172-222): out[j] = src[j + cut] inside [0, Lin), else 0
  const int W = cfg.in_samples;
  long long lo = 0, hi = W;                      // kept phases t: lo <= t - cut < hi
  if (cfg.p_position_ratio >= 0.0 && cfg.p_position_ratio <= 1.0) {
    const long long at = (long long)__dmul_rn((double)W, cfg.p_position_ratio);
    rec.cut = (int)((np > 0 ? p[0] : at) - at);  // an event without P (the reference raises) is cut from sample 0
  } else if (Lin > W) {
    long long m = Lin - W;
    for (int i = 0; i < np; ++i) m = p[i] < m ? p[i] : m;
    m -= gap;
    rec.cut = (int)r.randint(0, m > 1 ? m : 1);
  } else {
    if (Lin < W) rec.flags |= AUG_F_NORM64;      // the reference pads with float64 zeros and normalises in double
    lo = -(1ll << 40); hi = 1ll << 40;           // phases are kept as they are
  }
  int op = 0, os = 0;
  for (int i = 0; i < np; ++i) { const long long t = p[i] - rec.cut; if (t >= lo && t < hi) ppks_out[n * K_out + op++] = t; }
  for (int i = 0; i < ns; ++i) { const long long t = s[i] - rec.cut; if (t >= lo && t < hi) spks_out[n * K_out + os++] = t; }
  for (; op < K_out; ++op) ppks_out[n * K_out + op] = -10000000ll;
  for (; os < K_out; ++os) spks_out[n * K_out + os] = -10000000ll;
  cleared[n] = noise ? 1 : 0;
  rec_out[n] = rec;
}

// ---- apply ------------------------------------------------------------------------------------------------------------
__device__ double aug_block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < AUG_NT / 32; ++w) s += red[w];
  return s;
}
__device__ double aug_block_max(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = red[0];
  for (int w = 1; w < AUG_NT / 32; ++w) s = fmax(s, red[w]);
  return s;
}

__global__ void __launch_bounds__(AUG_NT) aug_apply_kernel(const float* __restrict__ data, int C, int Lin, SeistAugCfg cfg,
                                                           const uint64_t* __restrict__ seed_p, const AugRecipe* __restrict__ recs,
                                                           float* __restrict__ x) {
  extern __shared__ float s_x[];                 // (C, Lin), held in the reference's order before `shift`, see phys()
  __shared__ double red[AUG_NT / 32];
  __shared__ AugRecipe rec;
  const long long n = blockIdx.x;
  const int tid = threadIdx.x;
  if (tid == 0) rec = recs[n];
  const float* src = data + n * (long long)C * Lin;
  for (int i = tid; i < C * Lin; i += AUG_NT) s_x[i] = src[i];
  __syncthreads();
  const uint64_t seed = load_seed(seed_p);
  const int fl = rec.flags;
  // data after the roll of _shift_event at logical sample i sits at physical (i - shift) mod Lin
  const int shift = rec.shift;
  auto phys = [&](int i) { const int j = i - shift; return j < 0 ? j + Lin : j; };

  for (int f = 0; f < rec.n_fill; ++f)           // _generate_noise_data: randn over [P, coda end) of every pick pair
    for (int c = 0; c < C; ++c)
      for (int i = rec.fill_lo[f] + tid; i < rec.fill_hi[f]; i += AUG_NT)
        s_x[c * Lin + i] = (float)aug_normal(seed, AUG_STREAM_NORMAL + 0, aug_nidx(n, C, c, i));
  for (int a = 0; a < rec.n_add; ++a) {          // _add_event: source and target never overlap
    __syncthreads();
    const float sc = rec.add_scale[a];
    for (int c = 0; c < C; ++c)
      for (int i = tid; i < rec.add_len[a]; i += AUG_NT)
        s_x[c * Lin + rec.add_dst[a] + i] = __fadd_rn(s_x[c * Lin + rec.add_dst[a] + i], __fmul_rn(s_x[c * Lin + rec.add_src[a] + i], sc));
  }
  __syncthreads();
  if (fl & AUG_F_DROP) {                         // _drop_channel + _adjust_amplitude
    int nz = 0;
    for (int c = 0; c < C; ++c) {
      const bool dropped = (rec.drop_mask >> c) & 1;
      double m = 0.0;
      for (int i = tid; i < Lin; i += AUG_NT) {
        if (dropped) s_x[c * Lin + i] = 0.f;
        else m = fmax(m, (double)fabsf(s_x[c * Lin + i]));
      }
      nz += aug_block_max(m, red) > 0.0;
    }
    if (nz > 0) {
      const double f = (double)C / (double)nz;
      for (int i = tid; i < C * Lin; i += AUG_NT) s_x[i] = (float)__dmul_rn((double)s_x[i], f);
    }
    __syncthreads();
  }
  if (fl & (AUG_F_SCALE_MUL | AUG_F_SCALE_DIV)) {
    const float sc = rec.scale;
    const bool mul = fl & AUG_F_SCALE_MUL;
    for (int i = tid; i < C * Lin; i += AUG_NT) s_x[i] = mul ? __fmul_rn(s_x[i], sc) : __fdiv_rn(s_x[i], sc);
    __syncthreads();
  }
  if (fl & AUG_F_PRE) {                          // y[i] = x[i] - fl32(ratio) x[i-1], i >= 1; tiles from the end
    const float a = cfg.pre_emphasis_ratio;
    for (int c = 0; c < C; ++c) {
      float* row = s_x + c * Lin;
      for (int base = ((Lin - 1) / AUG_NT) * AUG_NT; base >= 0; base -= AUG_NT) {
        const int i = base + tid;
        const bool in = i >= 1 && i < Lin;
        const float y = in ? __fsub_rn(row[phys(i)], __fmul_rn(a, row[phys(i - 1)])) : 0.f;
        __syncthreads();
        if (in) row[phys(i)] = y;
        __syncthreads();
      }
    }
  }
  if (fl & AUG_F_NOISE) {                        // per-channel power in float32, the noise in float64
    for (int c = 0; c < C; ++c) {
      double q = 0.0;
      for (int i = tid; i < Lin; i += AUG_NT) { const float v = s_x[c * Lin + i]; q += (double)__fmul_rn(v, v); }
      const float px = (float)(aug_block_sum(q, red) / (double)Lin);
      const float pn = __fmul_rn(px, (float)exp10(-(double)rec.snr[c] / 10.0));
      const double amp = (double)__fsqrt_rn(pn);
      for (int i = tid; i < Lin; i += AUG_NT) {
        const int j = c * Lin + phys(i);
        s_x[j] = (float)__dadd_rn((double)s_x[j], __dmul_rn(aug_normal(seed, AUG_STREAM_NORMAL + 1, aug_nidx(n, C, c, i)), amp));
      }
    }
    __syncthreads();
  }
  if (fl & AUG_F_GAP) {
    for (int c = 0; c < C; ++c)
      for (int i = rec.gap_lo + tid; i < rec.gap_hi; i += AUG_NT) s_x[c * Lin + phys(i)] = 0.f;
    __syncthreads();
  }
  const int ws = cfg.window;
  if (fl & (AUG_F_MASKW | AUG_F_NOISEW)) {      // mask windows (value 1), then noise windows (randn)
    const int nw = Lin / ws;
    for (int i = tid; i < nw * ws; i += AUG_NT) {
      const int w = i / ws;
      const bool nzw = (fl & AUG_F_NOISEW) && ((rec.noise_bits[w >> 5] >> (w & 31)) & 1u);
      const bool mkw = (fl & AUG_F_MASKW) && ((rec.mask_bits[w >> 5] >> (w & 31)) & 1u);
      for (int c = 0; c < C; ++c) {
        if (nzw) s_x[c * Lin + phys(i)] = (float)aug_normal(seed, AUG_STREAM_NORMAL + 2, aug_nidx(n, C, c, i));
        else if (mkw) s_x[c * Lin + phys(i)] = 1.f;
      }
    }
    __syncthreads();
  }
  // _cut_window + _normalize (:224-242) per channel over the W-sample window
  const int W = cfg.in_samples, cut = rec.cut;
  const bool d64 = fl & AUG_F_NORM64;
  float* out = x + n * (long long)C * W;
  for (int c = 0; c < C; ++c) {
    const float* row = s_x + c * Lin;
    auto val = [&](int j) { const int i = j + cut; return (i >= 0 && i < Lin) ? row[phys(i)] : 0.f; };
    double sum = 0.0;
    for (int j = tid; j < W; j += AUG_NT) sum += (double)val(j);
    const double mean_d = aug_block_sum(sum, red) / (double)W;
    const float mean_f = (float)mean_d;
    double scale = 1.0;
    if (cfg.norm_mode == 1) {
      double q = 0.0;
      for (int j = tid; j < W; j += AUG_NT) {
        const double dv = d64 ? (double)val(j) - mean_d : (double)(val(j) - mean_f);
        q += dv * dv;
      }
      scale = sqrt(aug_block_sum(q, red) / (double)W);
      if (!d64) scale = (double)(float)scale;
    } else if (cfg.norm_mode == 2) {
      double m = -INFINITY;
      for (int j = tid; j < W; j += AUG_NT) m = fmax(m, d64 ? (double)val(j) - mean_d : (double)(val(j) - mean_f));
      scale = aug_block_max(m, red);
    }
    if (scale == 0.0) scale = 1.0;
    const float scale_f = (float)scale;
    for (int j = tid; j < W; j += AUG_NT)
      out[c * W + j] = d64 ? (float)(((double)val(j) - mean_d) / scale) : (float)__fdiv_rn(val(j) - mean_f, scale_f);
    __syncthreads();
  }
}

}  // namespace seist

using namespace seist;

extern "C" {

uint64_t seist_sizeof_aug(void) { return sizeof(SeistAugCfg); }

int seist_augment(const float* data, int64_t N, int32_t C, int32_t Lin, const int64_t* ppks, const int64_t* spks, int32_t K,
                  const double* snr, int32_t S, const uint8_t* augment, const SeistAugCfg* cfg, const uint64_t* seed,
                  float* x, int64_t* ppks_out, int64_t* spks_out, int32_t K_out, uint8_t* cleared, void* work,
                  int64_t work_bytes, void* stream) {
  if (!data || !ppks || !spks || !cfg || !seed || !x || !ppks_out || !spks_out || !cleared || !work || N <= 0 || C < 1 ||
      C > AUG_MAXC || Lin < 3 || Lin > 16384 || K < 1 || K_out < K || K_out > AUG_MAXK || S < 0 || (S > 0 && !snr)) {
    set_error("augment: bad arguments (1 <= C <= 8, 3 <= Lin <= 16384, 1 <= K <= K_out <= 8)");
    return -1;
  }
  const SeistAugCfg c = *cfg;
  if (c.in_samples < 1 || c.window < 1 || c.norm_mode < 0 || c.norm_mode > 2 || c.max_event_num > AUG_MAXK ||
      (c.add_event_rate > 0.0 && c.max_event_num > K_out) ||
      ((c.mask_percent > 0 || c.noise_percent > 0) && Lin / c.window > AUG_MAXWIN)) {
    set_error("augment: bad configuration (norm mode 0..2, max_event_num <= K_out, at most 1024 mask / noise windows)");
    return -1;
  }
  if (work_bytes < N * (int64_t)sizeof(AugRecipe)) { set_error("augment: workspace too small"); return -1; }
  const size_t smem = (size_t)C * Lin * sizeof(float);
  static size_t attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    const cudaError_t e = cudaFuncSetAttribute(aug_apply_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("augment: trace does not fit in shared memory"); return (int)e; }
    attr = smem;
  }
  cudaStream_t s = (cudaStream_t)stream;
  AugRecipe* rec = (AugRecipe*)work;
  aug_draw_kernel<<<(unsigned)((N + AUG_DRAW_NT - 1) / AUG_DRAW_NT), AUG_DRAW_NT, 0, s>>>(
      (const long long*)ppks, (const long long*)spks, K, snr, S, augment, N, C, Lin, c, seed, rec, (long long*)ppks_out,
      (long long*)spks_out, K_out, cleared);
  note_launch();
  if (int rc = check_launch("aug_draw")) return rc;
  aug_apply_kernel<<<(unsigned)N, AUG_NT, smem, s>>>(data, C, Lin, c, seed, rec, x);
  note_launch();
  return check_launch("aug_apply");
}

int seist_aug_recipe_bytes(void) { return (int)sizeof(AugRecipe); }

}  // extern "C"
