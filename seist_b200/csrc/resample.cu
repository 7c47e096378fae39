// Polyphase resampling of continuous records to the model's sampling rate (DESIGN §4.24): scipy.signal.resample_poly(x, up,
// down, axis=-1) with its defaults (Kaiser(5.0) anti-aliasing filter, zeros outside the record), for whole records and for
// streams pushed in chunks.  Output k lies at input time k * down / up and is
//   y[k] = sum over the in-record inputs i of x[i] * h[k * down - i * up + hl],  0 <= k * down - i * up + hl <= 2 * hl,
// hl = 10 * max(up, down), h the 2 * hl + 1 taps designed on the host (seist_b200/resample.py).  Inputs outside the record
// are skipped rather than multiplied by a zero, so a NaN input makes NaN exactly the outputs whose support holds it.
#include <algorithm>

#include "common.cuh"

namespace seist {

constexpr int RS_NT = 256;
constexpr int RS_TILE = 1024;      // outputs per CTA, halved while the tile's staged input span exceeds RS_SPAN
constexpr int RS_SPAN = 16384;     // staged input floats per CTA at most (64 KB)
constexpr int RS_MAX_RATE = 256;

struct RsFilter {
  int up, down, hl, nt;            // nt = taps of the longest phase (phase 0) = 2 * hl / up + 1
};

inline RsFilter rs_filter(int up, int down) {
  RsFilter f{up, down, 10 * std::max(up, down), 0};
  f.nt = 2 * f.hl / up + 1;
  return f;
}

// inputs a tile of `tile` outputs reads at most
inline long long rs_span(const RsFilter& f, int tile) { return ((long long)(tile - 1) * f.down + 2LL * f.hl) / f.up + 1; }

inline int rs_tile(const RsFilter& f) {
  int t = RS_TILE;
  while (t > 1 && rs_span(f, t) > RS_SPAN) t /= 2;
  return t;
}

__host__ __device__ inline int rs_taps_pad(const RsFilter& f) { return (f.up * f.nt + 3) & ~3; }

__host__ __device__ __forceinline__ long long rs_ceil_div(long long a, long long b) { return a >= 0 ? (a + b - 1) / b : -((-a) / b); }

// One stream call (or a whole record): row r = (station r / C, channel r % C).
struct RsCall {
  const float* src;          // whole record: the record; stream: the held inputs.  Row r at src + r * ld
  long long ld;
  const float* chunk;        // stream: the push, station s a (C, n_s) block at C * chunk_off[s]
  long long chunk_cap;
  const int64_t* desc;       // stream: N0, lo0, K0, lo1 (S each), chunk_off, out_off (S + 1 each); null for a whole record
  long long T, T_out;        // whole record
  float* out;                // whole record: (rows, T_out); stream: station s a (C, m_s) block at C * out_off[s]
  long long out_cap;
  float* held_out;           // stream: the new held inputs, same layout as src
  int S, C, tiles, tile;
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

__global__ void __launch_bounds__(RS_NT) resample_kernel(RsCall p, const float* __restrict__ taps_g, RsFilter f) {
  extern __shared__ __align__(16) float rs_smem[];
  const long long row = blockIdx.x / p.tiles;
  const int tile = (int)(blockIdx.x % p.tiles);
  // the row's inputs: [lo0, N0) held (the record: lo0 = 0, N0 = T), then [N0, N) from the push; outputs K0 .. K0 + m - 1
  long long N0, lo0 = 0, n_new = 0, K0 = 0, m, lo1 = 0;
  const float* held = p.src + row * p.ld;
  const float* chunk = p.chunk;
  float* dst;
  if (!p.desc) {
    N0 = p.T;
    m = p.T_out;
    dst = p.out + row * p.T_out;
  } else {
    const long long S = p.S, s = row / p.C, c = row % p.C;
    const int64_t* coff = p.desc + 4 * S;
    const int64_t* ooff = coff + S + 1;
    N0 = p.desc[s];
    lo0 = p.desc[S + s];
    K0 = p.desc[2 * S + s];
    lo1 = p.desc[3 * S + s];
    n_new = coff[s + 1] - coff[s];
    m = ooff[s + 1] - ooff[s];
    // a malformed descriptor gives wrong output but no out-of-range access
    if (lo0 < 0 || N0 < lo0 || N0 - lo0 > p.ld || K0 < 0 || n_new < 0 || coff[s] < 0 || p.C * coff[s + 1] > p.chunk_cap || m < 0 ||
        ooff[s] < 0 || p.C * ooff[s + 1] > p.out_cap || lo1 < lo0 || N0 + n_new - lo1 > p.ld)
      return;
    chunk += p.C * coff[s] + c * n_new;
    dst = p.out + p.C * ooff[s] + c * m;
  }
  const long long N = N0 + n_new;
  float* taps = rs_smem;
  float* xs = rs_smem + rs_taps_pad(f);
  const long long k0 = K0 + (long long)tile * p.tile, k1 = std::min(K0 + m, k0 + p.tile);
  long long gs = 0, ge = -1;
  if (k0 < k1) {
    rs_stage(taps, taps_g, (long long)f.up * f.nt);
    gs = std::max(rs_ceil_div(k0 * f.down - f.hl, f.up), lo0);
    ge = std::min(((k1 - 1) * f.down + f.hl) / f.up, N - 1);
    if (gs < N0) rs_stage(xs, held + (gs - lo0), std::min(ge + 1, N0) - gs);
    if (ge >= N0) rs_stage(xs + (std::max(gs, N0) - gs), chunk + (std::max(gs, N0) - N0), ge + 1 - std::max(gs, N0));
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    for (long long k = k0 + threadIdx.x; k < k1; k += RS_NT) dst[k - K0] = rs_output(xs, gs, ge, k, taps, f);
  }
  // stream: the inputs later outputs still read, [lo1, N), into the other held buffer
  if (p.desc && tile == 0) {
    float* keep = p.held_out + row * p.ld;
    for (long long j = threadIdx.x; j < N - lo1; j += RS_NT) {
      const long long g = lo1 + j;
      keep[j] = g < N0 ? held[g - lo0] : chunk[g - N0];
    }
  }
}

static int rs_launch(const RsCall& call, const float* taps, RsFilter f, long long rows, cudaStream_t stream, const char* what) {
  const long long grid = (long long)call.tiles * rows;
  if (grid > INT32_MAX) {
    set_error("resample: more than 2^31 - 1 CTAs (rows * output tiles)");
    return -1;
  }
  const int smem = (int)sizeof(float) * (rs_taps_pad(f) + (int)rs_span(f, call.tile));
  static int attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    cudaFuncSetAttribute(resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr = smem;
  }
  resample_kernel<<<(unsigned)grid, RS_NT, smem, stream>>>(call, taps, f);
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
  const RsFilter f = rs_filter(up, down);
  RsCall c{};
  c.src = record;
  c.ld = T;
  c.T = T;
  c.T_out = rs_ceil_div(T * up, down);
  c.out = out;
  c.tile = rs_tile(f);
  c.tiles = (int)std::min<long long>(INT32_MAX, rs_ceil_div(c.T_out, c.tile));
  return rs_launch(c, taps, f, rows, (cudaStream_t)stream, "resample");
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
  const RsFilter f = rs_filter(up, down);
  RsCall c{};
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
  c.tile = rs_tile(f);
  c.tiles = (int)std::max<long long>(1, std::min<long long>(INT32_MAX, rs_ceil_div(max_m, c.tile)));
  return rs_launch(c, taps, f, (long long)S * C, (cudaStream_t)stream, "resample_stream");
}

}  // extern "C"
