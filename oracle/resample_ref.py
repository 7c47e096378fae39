"""CPU oracle (TEST INFRASTRUCTURE) for polyphase resampling (seist_b200/resample.py, DESIGN §4.24), in float64.

  * `taps`     — scipy.signal.firwin(2 * hl + 1, 1 / max(up, down), window=('kaiser', 5.0)) * up, hl = 10 * max(up, down),
                 as resample_poly designs it: a windowed sinc normalised to unit DC gain;
  * `resample` — resample_poly(x, up, down, axis=-1) with zeros outside the record, restated directly: output k of a row of
                 T inputs, k < ceil(T * up / down), is the sum over the inputs 0 <= i < T with 0 <= k * down - i * up + hl
                 <= 2 * hl of x[i] * h[k * down - i * up + hl].  Inputs outside the record are skipped, so a NaN input makes
                 NaN exactly the outputs whose support holds it;
  * `StreamRef` — the same outputs emitted as a stream: after N inputs output k is final when k < ceil(N * up / down) and
                 k * down + hl < N * up, the close makes the rest final, and a station holds only the inputs from
                 ceil((K * down - hl) / up) (clipped to [0, N]) on, K its outputs so far: at most (2 * hl + down) // up + 1.
                 up == down passes every sample through as it arrives.
"""
import math

import numpy as np


def ratio(input_rate: int, output_rate: int):
    g = math.gcd(input_rate, output_rate)
    return output_rate // g, input_rate // g


def taps(up: int, down: int) -> np.ndarray:
    L = max(up, down)
    hl = 10 * L
    M = 2 * hl + 1
    h = np.sinc((np.arange(M) - hl) / L) / L * np.kaiser(M, 5.0)
    return h / h.sum() * up


def _ceil_div(a, b):
    return -((-a) // b)


def outputs(x: np.ndarray, g0: int, N: int, k0: int, k1: int, up: int, down: int) -> np.ndarray:
    """Outputs k0 .. k1 - 1 of rows whose inputs 0 .. N - 1 are known, x[..., j] holding input g0 + j (every input those
    outputs read from [0, N)), summed over the tap index in ascending order."""
    h = taps(up, down)
    hl = 10 * max(up, down)
    k = np.arange(k0, k1, dtype=np.int64)
    y = np.zeros(x.shape[:-1] + (k.size,))
    for j in range(2 * hl + 1):
        num = k * down + hl - j
        i = num // up
        ok = (num % up == 0) & (i >= 0) & (i < N)
        if ok.any():
            y[..., ok] += x[..., i[ok] - g0] * h[j]
    return y


def resample(x: np.ndarray, up: int, down: int) -> np.ndarray:
    """resample_poly(x, up, down, axis=-1) of float64 rows x (..., T)."""
    x = np.asarray(x, dtype=np.float64)
    if up == down:
        return x.copy()
    T = x.shape[-1]
    return outputs(x, 0, T, 0, _ceil_div(T * up, down), up, down)


class StreamRef:
    """S stations of C channels resampled as their samples arrive: `push(chunks)` (S float64 (C, n_s) arrays) and `close()`
    return each station's newly final outputs as a list of (C, m_s) arrays; `calls` records each call's N0, lo0, K0, lo1,
    N1, K1 per station."""

    def __init__(self, S: int, C: int, up: int, down: int):
        self.S, self.C, self.up, self.down = S, C, up, down
        self.hl = 10 * max(up, down)
        self.bound = (2 * self.hl + down) // up + 1
        self.N = np.zeros(S, np.int64)
        self.K = np.zeros(S, np.int64)
        self.lo = np.zeros(S, np.int64)
        self.held = [np.zeros((C, 0)) for _ in range(S)]
        self.calls = []
        self.closed = False

    def push(self, chunks):
        return self._call(chunks, False)

    def close(self):
        return self._call([np.zeros((self.C, 0))] * self.S, True)

    def _call(self, chunks, close: bool):
        assert not self.closed
        u, d, hl = self.up, self.down, self.hl
        outs, rec = [], {k: np.zeros(self.S, np.int64) for k in ("N0", "lo0", "K0", "lo1", "N1", "K1")}
        for s, c in enumerate(chunks):
            seq = np.concatenate([self.held[s], np.asarray(c, dtype=np.float64)], axis=1)
            N1 = int(self.N[s]) + c.shape[1]
            K1 = _ceil_div(N1 * u, d)
            if not close:
                K1 = min(K1, max(0, _ceil_div(N1 * u - hl, d)))
            K0, lo0 = int(self.K[s]), int(self.lo[s])
            if u == d:                                       # the identity passes every sample through at once
                K1 = lo1 = N1
                y = seq.copy()
            else:
                y = outputs(seq, lo0, N1, K0, K1, u, d)
                lo1 = min(max(_ceil_div(K1 * d - hl, u), 0), N1)
            outs.append(y)
            self.held[s] = seq[:, lo1 - lo0:]
            assert self.held[s].shape[1] <= self.bound
            for k, v in zip(rec, (self.N[s], lo0, K0, lo1, N1, K1)):
                rec[k][s] = v
            self.N[s], self.K[s], self.lo[s] = N1, K1, lo1
        self.calls.append(rec)
        self.closed = close
        return outs
