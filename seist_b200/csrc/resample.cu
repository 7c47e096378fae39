// Polyphase resampling of continuous records to the model's sampling rate (DESIGN §4.24): scipy.signal.resample_poly(x, up,
// down, axis=-1) with its defaults (Kaiser(5.0) anti-aliasing filter, zeros outside the record), for whole records and for
// streams pushed in chunks.  Output k lies at input time k * down / up and is
//   y[k] = sum over the in-record inputs i of x[i] * h[k * down - i * up + hl],  0 <= k * down - i * up + hl <= 2 * hl,
// hl = 10 * max(up, down), h the 2 * hl + 1 taps designed on the host (seist_b200/resample.py).  Inputs outside the record
// are skipped rather than multiplied by a zero, so a NaN input makes NaN exactly the outputs whose support holds it.
#include <algorithm>
#include <cstring>

#include "common.cuh"

namespace seist {

constexpr int RS_NT = 256;
constexpr int RS_TILE = 1024;      // outputs per CTA, halved while the tile's staged input span exceeds RS_SPAN
constexpr int RS_SPAN = 16384;     // staged input floats per CTA at most (64 KB)
constexpr int RS_MAX_RATE = 256;

// One filter: a row of the filter table (int32 x 8, seist_resample_table).  An identity row (up == down) has hl = nt = 0 and
// no taps: its outputs are its inputs, copied bit for bit.
struct RsFilter {
  int up, down, hl, nt;            // nt = taps of the longest phase (phase 0) = 2 * hl / up + 1
  int tap_off, tile, identity, smem;   // first tap in the concatenated table, outputs per CTA, dynamic shared bytes it needs
};
static_assert(sizeof(RsFilter) == 8 * sizeof(int32_t), "RsFilter is one row of the filter table");

// inputs a tile of `tile` outputs reads at most
__host__ __device__ inline long long rs_span(const RsFilter& f, int tile) {
  return ((long long)(tile - 1) * f.down + 2LL * f.hl) / f.up + 1;
}

inline int rs_tile(const RsFilter& f) {
  int t = RS_TILE;
  while (t > 1 && rs_span(f, t) > RS_SPAN) t /= 2;
  return t;
}

__host__ __device__ inline int rs_taps_pad(const RsFilter& f) { return (f.up * f.nt + 3) & ~3; }

__host__ __device__ inline int rs_smem(const RsFilter& f) { return (int)sizeof(float) * (rs_taps_pad(f) + (int)rs_span(f, f.tile)); }

// the filter seist_resample and seist_resample_stream apply: hl = 10 * max(up, down) even at up == down
inline RsFilter rs_filter(int up, int down) {
  RsFilter f{up, down, 10 * std::max(up, down), 0, 0, 0, 0, 0};
  f.nt = 2 * f.hl / up + 1;
  f.tile = rs_tile(f);
  f.smem = rs_smem(f);
  return f;
}

__host__ __device__ __forceinline__ long long rs_ceil_div(long long a, long long b) { return a >= 0 ? (a + b - 1) / b : -((-a) / b); }

// One call: a whole record or a stream call, of one filter or of a filter table.  Row r = (station r / C, channel r % C).
struct RsCall {
  const float* src;          // whole record of one filter: the record; stream: the held inputs.  Row r at src + r * ld
  long long ld;
  const float* chunk;        // stream: the push, station s a (C, n_s) block at C * chunk_off[s]
  long long chunk_cap;
  const int64_t* desc;       // stream: N0, lo0, K0, lo1 (S each), chunk_off, out_off (S + 1 each) [, filt (S), cta_off (S + 1)];
                             // whole record of a table: src, T, filt (S each), cta_off (S + 1); null for a whole record of one filter
  long long T, T_out;        // whole record: T (one filter) and the output row stride
  float* out;                // whole record: (rows, T_out); stream: station s a (C, m_s) block at C * out_off[s]
  long long out_cap;
  float* held_out;           // stream: the new held inputs, same layout as src
  const RsFilter* table;     // null: every row applies f over `tiles` CTAs; else station s applies table[filt[s]] over CTAs
  RsFilter f;                // cta_off[s] .. cta_off[s + 1] - 1, C per tile
  int F, S, C, tiles;
  bool stream;
};
// Output k of a row whose inputs gs .. ge are staged at xs[i - gs]: x[i] * h[k * down - i * up + hl] over the in-record
// inputs in ascending i, one fmaf each, accumulated in fp32.  Every path (whole records and every stream call) computes every
// output here from the same inputs, so a stream's outputs are bit-identical to the whole record's.  The taps are phase-major:
// phase phi = (k * down + hl) mod up holds h[phi + (nt_phi - 1 - t) * up] at taps[phi * nt + t], the order of ascending i.
__device__ __forceinline__ float rs_output(const float* xs, long long gs, long long ge, long long k, const float* taps, RsFilter f) {
  const long long a = k * f.down + f.hl;
  const long long ihi = a / f.up;
  const int phi = (int)(a - ihi * f.up);
  const long long ilo = ihi - (2 * f.hl - phi) / f.up;
  const long long i0 = max(ilo, gs), i1 = min(ihi, ge);
  const float* h = taps + (long long)phi * f.nt + (i0 - ilo);
  const float* x = xs + (i0 - gs);
  const int n = (int)(i1 - i0 + 1);
  float acc = 0.0f;
  for (int j = 0; j < n; ++j) acc = __fmaf_rn(x[j], h[j], acc);
  return acc;
}

// cp.async n floats global -> shared: 16-byte copies where source and destination share their alignment, 4-byte ones elsewhere
__device__ __forceinline__ void rs_stage(float* dst, const float* src, long long n) {
  const uint32_t d = smem_addr(dst);
  long long head = n;
  if (((uint32_t)(uintptr_t)src & 15u) == (d & 15u)) head = std::min<long long>(n, ((16u - (d & 15u)) & 15u) / 4);
  const long long nv = (n - head) / 4;
  for (long long j = threadIdx.x; j < head; j += RS_NT) cp_async4(d + 4 * (uint32_t)j, src + j);
  for (long long j = threadIdx.x; j < nv; j += RS_NT) cp_async16(d + 4 * (uint32_t)(head + 4 * j), src + head + 4 * j);
  for (long long j = head + 4 * nv + threadIdx.x; j < n; j += RS_NT) cp_async4(d + 4 * (uint32_t)j, src + j);
}

// TABLE: station s applies p.table[filt[s]] and owns CTAs cta_off[s] .. (mixed rates); else every row applies p.f over
// p.tiles CTAs.  One body: the one-filter instance leaves out the lookup and the NaN tail, and keeps its 64 registers.
template <bool TABLE>
__global__ void __launch_bounds__(RS_NT) resample_kernel(RsCall p, const float* __restrict__ taps_g) {
  extern __shared__ __align__(16) float rs_smem_buf[];
  const long long S = p.S;
  long long s, c, tile, tiles = p.tiles;
  RsFilter f = p.f;
  if constexpr (!TABLE) {
    s = blockIdx.x / tiles / p.C;
    c = blockIdx.x / tiles % p.C;
    tile = blockIdx.x % tiles;
  } else {
    // the station whose CTA range holds this CTA: cta_off[s] <= blockIdx.x < cta_off[s + 1]
    const int64_t* filt = p.desc + (p.stream ? 6 * S + 2 : 2 * S);
    const int64_t* cta = filt + S;
    const long long b = blockIdx.x;
    long long lo = 0, hi = S - 1;
    while (lo < hi) {
      const long long mid = (lo + hi + 1) / 2;
      if (cta[mid] <= b) lo = mid; else hi = mid - 1;
    }
    s = lo;
    const long long fi = filt[s], per = cta[s + 1] - cta[s];
    // a malformed descriptor gives wrong output but no out-of-range access
    if (b < cta[s] || b >= cta[s + 1] || fi < 0 || fi >= p.F || per % p.C) return;
    f = p.table[fi];
    tiles = per / p.C;
    c = (b - cta[s]) / tiles;
    tile = (b - cta[s]) % tiles;
  }
  const long long row = s * p.C + c;
  // the row's inputs: [lo0, N0) held (the record: lo0 = 0, N0 = T), then [N0, N) from the push; outputs K0 .. K0 + m - 1
  long long N0, lo0 = 0, n_new = 0, K0 = 0, m, lo1 = 0;
  const float* held = p.src + row * p.ld;
  const float* chunk = p.chunk;
  float* dst;
  if (!p.stream) {
    N0 = p.T;
    if constexpr (TABLE) {
      N0 = p.desc[S + s];
      held = reinterpret_cast<const float*>(p.desc[s]) + c * N0;
    }
    m = rs_ceil_div(N0 * f.up, f.down);
    dst = p.out + row * p.T_out;
    if constexpr (TABLE) {
      if (N0 < 0 || m > p.T_out) return;
      // the CTAs past the row's output tiles fill its tail m .. T_out - 1 with NaN, each an equal share
      const long long tiles_out = rs_ceil_div(m, f.tile);
      if (tile >= tiles_out) {
        const long long fills = tiles - tiles_out, j = tile - tiles_out, tail = p.T_out - m;
        for (long long k = m + tail * j / fills + threadIdx.x; k < m + tail * (j + 1) / fills; k += RS_NT) dst[k] = __int_as_float(0x7fc00000);
        return;
      }
    }
  } else {
    const int64_t* coff = p.desc + 4 * S;
    const int64_t* ooff = coff + S + 1;
    N0 = p.desc[s];
    lo0 = p.desc[S + s];
    K0 = p.desc[2 * S + s];
    lo1 = p.desc[3 * S + s];
    n_new = coff[s + 1] - coff[s];
    m = ooff[s + 1] - ooff[s];
    if (lo0 < 0 || N0 < lo0 || N0 - lo0 > p.ld || K0 < 0 || n_new < 0 || coff[s] < 0 || p.C * coff[s + 1] > p.chunk_cap || m < 0 ||
        ooff[s] < 0 || p.C * ooff[s + 1] > p.out_cap || lo1 < lo0 || N0 + n_new - lo1 > p.ld)
      return;
    chunk += p.C * coff[s] + c * n_new;
    dst = p.out + p.C * ooff[s] + c * m;
  }
  const long long N = N0 + n_new;
  if constexpr (TABLE) {
    uint32_t smem_bytes;
    asm("mov.u32 %0, %%dynamic_smem_size;" : "=r"(smem_bytes));
    if (f.smem < 0 || (uint32_t)f.smem > smem_bytes) return;
  }
  float* taps = rs_smem_buf;
  float* xs = rs_smem_buf + rs_taps_pad(f);
  const long long k0 = K0 + tile * f.tile, k1 = std::min(K0 + m, k0 + f.tile);
  long long gs = 0, ge = -1;
  if (k0 < k1) {
    rs_stage(taps, taps_g + f.tap_off, (long long)f.up * f.nt);
    gs = std::max(rs_ceil_div(k0 * f.down - f.hl, f.up), lo0);
    ge = std::min(((k1 - 1) * f.down + f.hl) / f.up, N - 1);
    if (gs < N0) rs_stage(xs, held + (gs - lo0), std::min(ge + 1, N0) - gs);
    if (ge >= N0) rs_stage(xs + (std::max(gs, N0) - gs), chunk + (std::max(gs, N0) - N0), ge + 1 - std::max(gs, N0));
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    if (TABLE && f.identity)
      for (long long k = k0 + threadIdx.x; k < k1; k += RS_NT) dst[k - K0] = xs[k - gs];
    else
      for (long long k = k0 + threadIdx.x; k < k1; k += RS_NT) dst[k - K0] = rs_output(xs, gs, ge, k, taps, f);
  }
  // stream: the inputs later outputs still read, [lo1, N), into the other held buffer
  if (p.stream && tile == 0) {
    float* keep = p.held_out + row * p.ld;
    for (long long j = threadIdx.x; j < N - lo1; j += RS_NT) {
      const long long g = lo1 + j;
      keep[j] = g < N0 ? held[g - lo0] : chunk[g - N0];
    }
  }
}

static int rs_launch(const RsCall& call, const float* taps, long long ctas, int smem, cudaStream_t stream, const char* what) {
  if (ctas > INT32_MAX) {
    set_error("resample: more than 2^31 - 1 CTAs (rows * output tiles)");
    return -1;
  }
  const bool table = call.table != nullptr;
  static int attr[2] = {0, 0};
  if (smem > 48 * 1024 && smem > attr[table]) {
    cudaFuncSetAttribute(table ? resample_kernel<true> : resample_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr[table] = smem;
  }
  if (table)
    resample_kernel<true><<<(unsigned)ctas, RS_NT, smem, stream>>>(call, taps);
  else
    resample_kernel<false><<<(unsigned)ctas, RS_NT, smem, stream>>>(call, taps);
  note_launch();
  return check_launch(what);
}

static bool rs_rates_ok(int32_t up, int32_t down) { return up >= 1 && down >= 1 && up <= RS_MAX_RATE && down <= RS_MAX_RATE; }

}  // namespace seist

using namespace seist;

extern "C" {

int seist_resample(const float* record, int32_t rows, int64_t T, const float* taps, int32_t up, int32_t down, float* out, void* stream) {
  if (!record || !taps || !out || rows < 1 || T < 1 || T > (int64_t)1 << 40 || !rs_rates_ok(up, down)) {
    set_error("resample: bad arguments (non-null buffers, rows >= 1, 1 <= T <= 2^40, 1 <= up, down <= 256)");
    return -1;
  }
  RsCall c{};
  c.f = rs_filter(up, down);
  c.src = record;
  c.ld = T;
  c.T = T;
  c.T_out = rs_ceil_div(T * up, down);
  c.out = out;
  c.S = rows;
  c.C = 1;
  c.tiles = (int)std::min<long long>(INT32_MAX, rs_ceil_div(c.T_out, c.f.tile));
  return rs_launch(c, taps, (long long)c.tiles * rows, c.f.smem, (cudaStream_t)stream, "resample");
}

int seist_resample_stream(const float* held, int64_t H, const float* chunk, int64_t chunk_capacity, const int64_t* desc, int32_t S,
                          int32_t C, int64_t max_m, const float* taps, int32_t up, int32_t down, float* out, int64_t out_capacity,
                          float* held_out, void* stream) {
  if (!held || !chunk || !desc || !taps || !out || !held_out || held_out == held || S < 1 || C < 1 || H < 1 || chunk_capacity < 0 ||
      out_capacity < 0 || max_m < 0 || max_m > (int64_t)1 << 40 || !rs_rates_ok(up, down)) {
    set_error("resample_stream: bad arguments (non-null buffers, held_out distinct from held, S, C, H >= 1, 0 <= max_m <= 2^40, "
              "capacities >= 0, 1 <= up, down <= 256)");
    return -1;
  }
  RsCall c{};
  c.f = rs_filter(up, down);
  c.src = held;
  c.ld = H;
  c.chunk = chunk;
  c.chunk_cap = chunk_capacity;
  c.desc = desc;
  c.out = out;
  c.out_cap = out_capacity;
  c.held_out = held_out;
  c.S = S;
  c.C = C;
  c.stream = true;
  c.tiles = (int)std::max<long long>(1, std::min<long long>(INT32_MAX, rs_ceil_div(max_m, c.f.tile)));
  return rs_launch(c, taps, (long long)c.tiles * S * C, c.f.smem, (cudaStream_t)stream, "resample_stream");
}

int seist_resample_table(int32_t F, const int32_t* up, const int32_t* down, int32_t* table) {
  if (F < 1 || !up || !down || !table) {
    set_error("resample_table: bad arguments (F >= 1, non-null arrays)");
    return -1;
  }
  long long tap_off = 0;
  for (int i = 0; i < F; ++i) {
    if (!rs_rates_ok(up[i], down[i])) {
      set_error("resample_table: every ratio needs 1 <= up, down <= 256");
      return -1;
    }
    RsFilter f = up[i] == down[i] ? RsFilter{1, 1, 0, 0, 0, RS_TILE, 1, 0} : rs_filter(up[i], down[i]);
    f.tap_off = (int)tap_off;
    f.smem = rs_smem(f);
    tap_off += rs_taps_pad(f);
    if (tap_off > INT32_MAX) {
      set_error("resample_table: more than 2^31 - 1 taps in all");
      return -1;
    }
    std::memcpy(table + 8 * i, &f, sizeof f);
  }
  return 0;
}

static bool rs_table_ok(const int32_t* table, int32_t F, int32_t smem) {
  return table && F >= 1 && smem >= 0 && smem <= 227 * 1024;
}

int seist_resample_multi(const int64_t* desc, int32_t S, int32_t C, int64_t T_max, int64_t ctas, const int32_t* table, int32_t F,
                         int32_t smem, const float* taps, float* out, void* stream) {
  if (!desc || !taps || !out || S < 1 || C < 1 || T_max < 1 || T_max > (int64_t)1 << 40 || ctas < 1 || !rs_table_ok(table, F, smem)) {
    set_error("resample_multi: bad arguments (non-null buffers, S, C, ctas >= 1, 1 <= T_max <= 2^40, F >= 1, 0 <= smem <= 227 KB)");
    return -1;
  }
  RsCall c{};
  c.desc = desc;
  c.T_out = T_max;
  c.out = out;
  c.table = reinterpret_cast<const RsFilter*>(table);
  c.F = F;
  c.S = S;
  c.C = C;
  return rs_launch(c, taps, ctas, smem, (cudaStream_t)stream, "resample_multi");
}

int seist_resample_multi_stream(const float* held, int64_t H, const float* chunk, int64_t chunk_capacity, const int64_t* desc,
                                int32_t S, int32_t C, int64_t ctas, const int32_t* table, int32_t F, int32_t smem, const float* taps,
                                float* out, int64_t out_capacity, float* held_out, void* stream) {
  if (!held || !chunk || !desc || !taps || !out || !held_out || held_out == held || S < 1 || C < 1 || H < 1 || chunk_capacity < 0 ||
      out_capacity < 0 || ctas < 1 || !rs_table_ok(table, F, smem)) {
    set_error("resample_multi_stream: bad arguments (non-null buffers, held_out distinct from held, S, C, H, ctas >= 1, "
              "capacities >= 0, F >= 1, 0 <= smem <= 227 KB)");
    return -1;
  }
  RsCall c{};
  c.src = held;
  c.ld = H;
  c.chunk = chunk;
  c.chunk_cap = chunk_capacity;
  c.desc = desc;
  c.out = out;
  c.out_cap = out_capacity;
  c.held_out = held_out;
  c.table = reinterpret_cast<const RsFilter*>(table);
  c.F = F;
  c.S = S;
  c.C = C;
  c.stream = true;
  return rs_launch(c, taps, ctas, smem, (cudaStream_t)stream, "resample_multi_stream");
}

}  // extern "C"
