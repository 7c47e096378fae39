"""Seeded probability traces on which the pickers' tie rule decides the answer (tests/test_cpu_peak_ties.py,
tests/test_gpu_peak_ties.py, tests/golden/make_golden_peak_ties.py).

They hold what trace generators elsewhere rule out on purpose: values on a 2^-k grid, plateaus at exactly 1.0f and 0.9998f, equal-height
chains and clusters, values equal to float32(threshold), NaN next to candidates and at the row ends, rows without a
candidate.  `short_trace` is the fixture's input (L <= 8192); `long_rows` lays the same families out on rows of 2^20
samples at the picker kernels' size boundaries and returns where it put them.
"""
import numpy as np

F32 = np.float32
HEIGHTS = tuple(F32(v) for v in (1.0, 0.9998, 0.75, 0.7, 0.5, 0.3, 0.125))    # the tie-prone heights
THRESHOLDS = (0.7, 0.3)            # float32(0.7) < 0.7, float32(0.3) > 0.3: a value equal to float32(thr) is a pick (>=), not in a run (>)
LONG_T = 1 << 20
CL_SMALL, CL_SEG, CL_SMEM, ST_CH = 32, 1024, 4096, 4096     # csrc/stream.cu
GAP = 160                          # background between the motifs of a long row: > every min_peak_dist the tests use


def chain(n: int, spacing: int, h, trough=0.0) -> np.ndarray:
    """n candidates of height h, `spacing` samples apart, `trough` between them: (n - 1) * spacing + 1 samples."""
    out = np.full((n - 1) * spacing + 1, F32(trough), F32)
    out[::spacing] = F32(h)
    return out


def quantised(rng, n: int, bits: int) -> np.ndarray:
    """n values on the grid k / 2^bits, 0 <= k <= 2^bits (1.0 included)."""
    return (rng.integers(0, (1 << bits) + 1, n) / F32(1 << bits)).astype(F32)


def _motif(rng, mpd: int) -> np.ndarray:
    k = rng.integers(0, 7)
    h = HEIGHTS[rng.integers(0, len(HEIGHTS))]
    if k == 0:
        return quantised(rng, int(rng.integers(4, 300)), int(rng.integers(1, 5)))
    if k == 1:                                             # plateaus at 1.0 / 0.9998, close together
        h = HEIGHTS[rng.integers(0, 2)]
        parts = []
        for _ in range(rng.integers(2, 6)):
            parts += [np.full(rng.integers(1, 6), h, F32), np.full(rng.choice([1, 2, mpd, mpd + 1]), F32(rng.choice([0.0, 0.5])), F32)]
        return np.concatenate(parts)
    if k == 2:                                             # equal-height chain at spacing 2, mpd or mpd + 1
        return chain(int(rng.integers(2, 40)), int(rng.choice([2, mpd, mpd + 1])), h, rng.choice([0.0, 0.125]))
    if k == 3:                                             # an equal-height cluster around the one-thread limit
        return chain(int(rng.choice([CL_SMALL, CL_SMALL + 1])), 2, h)
    if k == 4:                                             # values equal to float32(threshold) next to larger ones
        v = np.array([0.0, 0.7, 0.0, 0.7, 0.7, 0.0, 0.3, 0.7, 0.3, 0.70000005, 0.7, 0.0], F32)
        return v[: rng.integers(3, v.size + 1)]
    if k == 5:                                             # NaN next to candidates
        v = quantised(rng, int(rng.integers(6, 60)), 3)
        v[rng.integers(0, v.size, max(1, v.size // 8))] = np.nan
        return v
    return np.full(rng.integers(1, 20), F32(rng.choice([0.0, 0.7, 1.0])), F32)       # flat: no candidate


def short_trace(seed: int, L: int, mpd: int, nan: bool) -> np.ndarray:
    """L float32 samples of motifs separated by random (often short) gaps, so that equal heights meet within mpd; with
    `nan`, NaN also next to random candidates and at samples 0, 1, L - 2, L - 1 (each with probability 1/2)."""
    rng = np.random.default_rng([seed, L, mpd, int(nan)])
    parts, n = [], 0
    while n < L:
        m = _motif(rng, mpd)
        if not nan:
            m = np.nan_to_num(m, nan=0.25)
        g = np.full(rng.choice([0, 1, 2, mpd - 1, mpd, mpd + 1, 3 * mpd]), F32(rng.choice([0.0, 0.125])), F32)
        parts += [m, g]
        n += m.size + g.size
    x = np.concatenate(parts)[:L].copy()
    if nan:
        c = candidates(x, 0.0)
        if c.size:
            pick = rng.choice(c, max(1, c.size // 10))
            x[np.clip(pick + rng.choice([-1, 1], pick.size), 0, L - 1)] = np.nan
        for i in (0, 1, L - 2, L - 1):
            if L > 1 and rng.integers(0, 2):
                x[i] = np.nan
    return x


def candidates(x: np.ndarray, mph: float) -> np.ndarray:
    """The rising-edge candidates of `_detect_peaks` (before the distance suppression): x[i] - x[i-1] > 0, x[i+1] - x[i] <= 0,
    x[i] >= mph, 0 < i < L - 1 (NaN comparisons are false, so NaN and its neighbours are never candidates)."""
    x = np.asarray(x, F32)
    if x.size < 3:
        return np.zeros(0, np.int64)
    with np.errstate(invalid="ignore"):
        i = np.nonzero((x[1:-1] - x[:-2] > 0) & (x[2:] - x[1:-1] <= 0) & (x[1:-1] >= F32(mph)))[0] + 1
    return i.astype(np.int64)


def cluster_last(x: np.ndarray, mph: float, mpd: int) -> dict:
    """Each candidate -> the last candidate of its cluster (consecutive candidates <= mpd apart)."""
    c = candidates(x, mph)
    out = {}
    j = 0
    while j < c.size:
        e = j
        while e + 1 < c.size and c[e + 1] - c[e] <= mpd:
            e += 1
        for k in range(j, e + 1):
            out[int(c[k])] = int(c[e])
        j = e + 1
    return out


class _Row:
    """A long row of background 0.0 that motifs are written into left to right, GAP samples apart."""

    def __init__(self, T):
        self.x = np.zeros(T, F32)
        self.at = 0
        self.marks = {}

    def put(self, m, name=None, at=None):
        a = self.at + GAP if at is None else at
        self.x[a:a + m.size] = m
        if name:
            self.marks[name] = a
        self.at = a + m.size
        return a


def long_rows(seed: int = 20261018, T: int = LONG_T):
    """Five (T,) float32 rows and, per row, the sample positions of its landmarks:
    row 0: equal candidates at 4095 and 4097 (the first ST_CH block of a whole row's candidate pass is samples 1 .. 4096),
           runs ending at 4095 and starting at 8192 (the run pass's blocks start at multiples of ST_CH), NaN at samples
           0, 1, T - 2, T - 1 with candidates beside them, equal chains at spacing 2, 3, 7, 8, 100, 101, clusters of 32 and
           33 equal candidates, plateaus at 1.0f and 0.9998f, float32(0.7) candidates and runs, NaN beside candidates;
    row 1: a cluster of 1023 equal candidates, then one of 40 that starts at candidate 1023 of the row and runs into the
           next CL_SEG, fillers up to candidate 2047, a cluster of 4097 (> CL_SMEM) starting there, one of 4096 (== CL_SMEM);
    row 2: a candidate at 4096, equal candidates at 8190, 8192, 8194, quantised noise at 2^-1 .. 2^-4;
    row 3: 0.8 everywhere: no candidate, one run over the whole row;
    row 4: 2^18 samples of 2^-2 noise (ties everywhere; with mpd = 100 one cluster of tens of thousands)."""
    rng = np.random.default_rng(seed)
    rows = [_Row(T) for _ in range(5)]
    r = rows[0]
    r.x[0:4] = (np.nan, np.nan, 0.9, 0.0)                 # 2 would be a candidate but for the NaN at 1
    r.x[4090:4096] = 0.8                                   # run [4090, 4095]; a candidate at 4090
    r.put(np.array([1.0, 0.0, 1.0], F32), "edge4095", at=4095)
    r.x[8192:8200] = 0.9                                   # run starting at 8192
    r.x[12280:12300] = 0.75                                # run across 12288
    r.at = 12300
    for sp in (2, 3, 7, 8, 100, 101):
        r.put(chain(12, sp, 0.9998), f"chain{sp}")
    r.put(chain(CL_SMALL, 2, 0.9998), "cluster32")
    r.put(chain(CL_SMALL + 1, 2, 1.0), "cluster33")
    for h in (1.0, 0.9998):
        for sep in (1, 2, 7, 8):
            m = np.concatenate([np.concatenate([np.full(w, h, F32), np.zeros(sep, F32)]) for w in (1, 2, 3, 4)])
            r.put(m, f"plateau{h}_{sep}")
    r.put(chain(5, 2, 0.7), "thr2")
    r.put(chain(3, 200, 0.7), "thr200")
    r.put(np.full(30, F32(0.7)), "thr_run")
    r.put(np.array([0.7, 0.70000005, 0.70000005, 0.7], F32), "thr_above")
    r.put(np.array([0.2, 0.9, np.nan, 0.3, np.nan, 0.9, 0.2, 0.9, np.nan, 0.9, 0.1], F32), "nan")
    for _ in range(20):
        r.put(quantised(rng, 3000, int(rng.integers(1, 5))))
        r.put(_nan_free(_motif(rng, 7)))
    r.x[T - 4:] = (0.0, 0.9, np.nan, np.nan)               # T - 3 would be a candidate but for the NaN at T - 2

    r = rows[1]
    r.put(chain(CL_SEG - 1, 2, 0.75), "prefix1023")
    r.put(chain(40, 2, 0.75), "seg_cross")                 # candidates 1023 .. 1062
    r.put(chain(2 * CL_SEG - 1 - (CL_SEG - 1) - 40, 2, 0.9))
    r.put(chain(CL_SMEM + 1, 2, 1.0), "cluster4097")       # starts at candidate 2047
    r.put(chain(CL_SMEM, 2, 0.9998), "cluster4096")
    for _ in range(30):
        r.put(_nan_free(_motif(rng, 7)))

    r = rows[2]
    r.x[4095:4098] = (0.0, 0.9, 0.0)
    r.marks["edge4096"] = 4096
    r.x[8189:8196] = (0.0, 0.9, 0.0, 0.9, 0.0, 0.9, 0.0)
    r.marks["edge8192"] = 8190
    r.at = 8196
    for bits in (1, 2, 3, 4):
        r.put(quantised(rng, 20_000, bits), f"noise{bits}")
    rows[3].x[:] = 0.8
    rows[4].put(quantised(rng, 1 << 18, 2), "noise", at=1000)
    return np.stack([r.x for r in rows]), [r.marks for r in rows]


def _nan_free(m):
    return np.nan_to_num(m, nan=0.25)


# the fixture tests/golden/reference_peak_ties.pt: every (mph, mpd, topk) of FIXTURE_PARAMS on every short trace of
# fixture_traces(); topk None is `_detect_peaks(topk=None)`
FIXTURE_PARAMS = ((0.7, 2, 3), (0.7, 7, 8), (0.3, 50, 5), (0.7, 2, None), (0.5, 5, None), (0.125, 7, None))
FIXTURE_L = (3, 4, 5, 64, 1000, 4096, 8192)
FIXTURE_SEEDS = 42


def fixture_traces(mpd: int):
    """(seed, L, nan, trace) of the fixture for one min_peak_dist: every L of FIXTURE_L six times, a third with NaN."""
    return [(s, FIXTURE_L[s % len(FIXTURE_L)], s % 3 == 2, short_trace(s, FIXTURE_L[s % len(FIXTURE_L)], mpd, s % 3 == 2))
            for s in range(FIXTURE_SEEDS)]
