"""Resampling continuous records and streams to the model's sampling rate on the device (DESIGN §4.24).

The shipped checkpoints are trained at their dataset's rate (DiTing: 50 Hz) and every annotator slices windows of
`in_samples` samples from what it is given, so a feed at another rate has to be converted first.  `Resampler` does that on
the GPU, equal to `scipy.signal.resample_poly(x, up, down, axis=-1)` with its defaults: up / down is output_rate /
input_rate reduced, the taps are firwin(2 * hl + 1, 1 / max(up, down), window=('kaiser', 5.0)) * up with hl = 10 * max(up,
down), zeros lie outside the record and a record of T samples gives ceil(T * up / down).  Output k lies at input time
k * down / up (sample 0 on sample 0), so picks downstream are indices at output_rate, and
`ContinuousAnnotator.from_args(..., sampling_rate=)` takes the model's rate, not the feed's.

A record (S, C, T) is one launch with no host synchronisation; `open_stream` streams stations chunk by chunk, each
station's concatenated output bit-identical to that of its whole record.  Non-finite samples are not special-cased: out-of-
record inputs are skipped rather than multiplied by zero, so an output is NaN exactly when a NaN input lies in its support,
and a gap widens by at most hl / up input samples on each side.  The float64 restatement is `oracle/resample_ref.py`.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import _lib

MAX_RATIO = 256          # largest up or down after reduction: at most 5 121 taps


def _s() -> int:
    return torch.cuda.current_stream().cuda_stream


def _prefix(counts) -> np.ndarray:
    return np.concatenate([[0], np.cumsum(counts, dtype=np.int64)]).astype(np.int64)


def _ceil_div(a, b):
    return -((-a) // b)


def design_taps(up: int, down: int) -> np.ndarray:
    """The float64 anti-aliasing filter of resample_poly(x, up, down): 2 * hl + 1 taps, hl = 10 * max(up, down), a Kaiser(5.0)
    windowed sinc with cutoff 1 / max(up, down) of the Nyquist rate, normalised to unit DC gain (firwin) and times up."""
    L = max(up, down)
    hl = 10 * L
    M = 2 * hl + 1
    c = 1.0 / L
    h = c * np.sinc(c * (np.arange(M) - hl)) * np.kaiser(M, 5.0)
    return h / h.sum() * up


def polyphase_taps(up: int, down: int) -> np.ndarray:
    """design_taps as the float32 (up, nt) table the kernel reads, nt = 2 * hl // up + 1: phase phi holds the taps of the
    outputs with (k * down + hl) % up == phi in the order of ascending input index, h[phi + (n - 1 - t) * up] at t < n =
    (2 * hl - phi) // up + 1, zeros after."""
    h = design_taps(up, down)
    hl = 10 * max(up, down)
    table = np.zeros((up, 2 * hl // up + 1))
    for phi in range(up):
        n = (2 * hl - phi) // up + 1
        table[phi, :n] = h[phi + (n - 1 - np.arange(n)) * up]
    return table.astype(np.float32)


def stream_plan(N, K, n, up: int, down: int, close: bool = False) -> dict:
    """One call of a resampling stream, per station, from its inputs received so far N (S,), outputs emitted so far K (S,)
    and this push's lengths n (S,) (ignored at the close).  After N1 inputs output k is final when k < ceil(N1 * up / down)
    and k * down + hl < N1 * up (every input with a nonzero tap has arrived); the close makes every k < ceil(N1 * up / down)
    final.  A station holds the inputs from lo = ceil((K * down - hl) / up) (clipped to [0, N]) on.  Returns int64 arrays
    N0, lo0, K0, lo1, N1, K1 (S,) and the exclusive prefixes chunk_off of the lengths and out_off of K1 - K0 (S + 1,)."""
    hl = 10 * max(up, down)
    N = np.asarray(N, dtype=np.int64).reshape(-1)
    K = np.asarray(K, dtype=np.int64).reshape(-1)
    n = np.zeros_like(N) if close else np.asarray(n, dtype=np.int64).reshape(-1)
    if n.shape != N.shape or (n < 0).any():
        raise ValueError(f"expected {N.size} non-negative lengths, got {n.tolist()}")
    N1 = N + n
    K1 = _ceil_div(N1 * up, down)
    if not close:
        K1 = np.minimum(K1, np.maximum(0, _ceil_div(N1 * up - hl, down)))

    def held_start(k, total):
        return np.clip(_ceil_div(k * down - hl, up), 0, total)
    return dict(N0=N, lo0=held_start(K, N), K0=K, lo1=held_start(K1, N1), N1=N1, K1=K1, chunk_off=_prefix(n), out_off=_prefix(K1 - K))


def _check_rate(v, what: str) -> int:
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or int(v) <= 0:
        raise ValueError(f"{what} must be a positive int, got {v!r}")
    return int(v)


class Resampler:
    """Resample (S, C, T) float32 records from input_rate to output_rate on `device` (positive ints; the ratio reduced by
    their gcd may have neither term above 256).  `rs(record)` -> (S, C, ceil(T * up / down)), equal to scipy's
    resample_poly(record, up, down, axis=-1) to fp32 accuracy; `open_stream(S)` -> a ResampleStream.  Stations of
    different input rates take one Resampler per rate."""

    def __init__(self, input_rate: int, output_rate: int, device="cuda"):
        fin, fout = _check_rate(input_rate, "input_rate"), _check_rate(output_rate, "output_rate")
        g = math.gcd(fin, fout)
        self.up, self.down = fout // g, fin // g
        if max(self.up, self.down) > MAX_RATIO:
            raise ValueError(f"{fin} -> {fout} Hz reduces to up {self.up}, down {self.down}: neither may exceed {MAX_RATIO}")
        self.input_rate, self.output_rate = fin, fout
        self.half_len = 10 * max(self.up, self.down)
        dev = torch.device(device)
        if dev.type != "cuda":
            raise ValueError(f"Resampler has no CPU path, got device {dev}")
        if dev.index is None and torch.cuda.is_available():
            dev = torch.device("cuda", torch.cuda.current_device())
        self.device = dev
        self.held_bound = (2 * self.half_len + self.down) // self.up + 1
        self._taps = None

    @property
    def identity(self) -> bool:
        return self.up == self.down

    def taps(self) -> torch.Tensor:
        """The polyphase table on the device, uploaded on first use."""
        if self._taps is None:
            self._taps = torch.from_numpy(polyphase_taps(self.up, self.down)).to(self.device)
        return self._taps

    def _check(self, t: torch.Tensor, what: str):
        if not torch.is_tensor(t) or t.dtype != torch.float32 or not t.is_cuda or t.device != self.device or not t.is_contiguous():
            got = f"{tuple(t.shape)} {t.dtype} on {t.device}" if torch.is_tensor(t) else type(t).__name__
            raise ValueError(f"{what}: expected a contiguous float32 CUDA tensor on {self.device}, got {got}")

    def __call__(self, record: torch.Tensor) -> torch.Tensor:
        if not torch.is_tensor(record) or record.dim() != 3 or min(record.shape) < 1:
            raise ValueError(f"expected a record (S, C, T) with S, C, T >= 1, got {tuple(record.shape) if torch.is_tensor(record) else record!r}")
        self._check(record, "record")
        S, C, T = record.shape
        if S * C > 2 ** 31 - 1:
            raise ValueError(f"at most 2^31 - 1 rows, got {S} x {C}")
        if self.identity:
            return record.clone()
        out = torch.empty(S, C, _ceil_div(T * self.up, self.down), device=self.device)
        _lib.check(_lib.lib().seist_resample(record.data_ptr(), S * C, T, self.taps().data_ptr(), self.up, self.down, out.data_ptr(), _s()),
                   "seist_resample")
        return out

    def open_stream(self, n_stations: int, channels: int = 3) -> "ResampleStream":
        return ResampleStream(self, n_stations, channels)


class ResampleStream:
    """A resampled stream of S stations of C channels (`Resampler.open_stream`).  `push(chunks)` takes an (S, C, n) tensor
    or a list of S (C, n_s) tensors (any n_s >= 0) and returns each station's newly final outputs in the same form: an
    (S, C, m) tensor or a list of S (C, m_s) tensors; a tensor push needs every station to have received as many samples.
    `close()` returns the rest, zeros past each station's end as in the
    whole record, in the form of the last push.  Per station, the concatenated outputs are bit-identical to `rs(record)` of
    its record.  Outputs lag the inputs by hl / up input samples (0.2 s at 100 -> 50 Hz).  Held between calls: N and K
    per station on the host and at most held_bound inputs per row in a fixed (S, C, held_bound) device buffer; a push reads
    nothing back from the device."""

    def __init__(self, rs: Resampler, n_stations: int, channels: int = 3):
        if int(n_stations) < 1 or int(channels) < 1:
            raise ValueError(f"need at least one station and one channel, got {n_stations}, {channels}")
        self.rs = rs
        self.S, self.C = int(n_stations), int(channels)
        self.held = [torch.zeros(self.S, self.C, rs.held_bound, device=rs.device) for _ in range(2)]
        self.N = np.zeros(self.S, np.int64)
        self.K = np.zeros(self.S, np.int64)
        self.closed = False
        self._as_list = False
        self._none = torch.zeros(1, device=rs.device)

    def push(self, chunks):
        if self.closed:
            raise RuntimeError("push() after close()")
        if torch.is_tensor(chunks):
            if chunks.dim() != 3 or tuple(chunks.shape[:2]) != (self.S, self.C):
                raise ValueError(f"expected an ({self.S}, {self.C}, n) chunk, got {tuple(chunks.shape)}")
            self.rs._check(chunks, "chunk")
            if (self.N != self.N[0]).any():
                raise ValueError(f"stations have received different numbers of samples {self.N.tolist()}: push a list of chunks")
            n = np.full(self.S, chunks.shape[2], np.int64)
            chunk, parts = chunks, None
        else:
            if len(chunks) != self.S:
                raise ValueError(f"expected {self.S} chunks (one per station), got {len(chunks)}")
            for s, c in enumerate(chunks):
                if not torch.is_tensor(c) or c.dim() != 2 or c.shape[0] != self.C:
                    raise ValueError(f"station {s}: expected a ({self.C}, n) chunk, got {tuple(c.shape) if torch.is_tensor(c) else c!r}")
                self.rs._check(c, f"station {s}")
            n = np.array([c.shape[1] for c in chunks], np.int64)
            parts = chunks
            chunk = torch.cat([c.reshape(-1) for c in chunks]) if n.sum() else self._none
        self._as_list = parts is not None
        if self.rs.identity:
            self.N += n
            self.K = self.N.copy()
            return [c.clone() for c in parts] if parts is not None else chunks.clone()
        return self._call(stream_plan(self.N, self.K, n, self.rs.up, self.rs.down), chunk if chunk.numel() else self._none)

    def close(self):
        if self.closed:
            raise RuntimeError("close() after close()")
        plan = stream_plan(self.N, self.K, None, self.rs.up, self.rs.down, close=True)
        if self.rs.identity:
            plan["out_off"][:] = 0
            plan["K1"] = self.K
        out = self._call(plan, self._none, launch=not self.rs.identity)
        self.closed = True
        return out

    def _call(self, plan: dict, chunk: torch.Tensor, launch: bool = True):
        rs, S, C = self.rs, self.S, self.C
        m = plan["K1"] - plan["K0"]
        off = plan["out_off"]
        out = torch.empty(max(1, C * int(off[-1])), device=rs.device)
        if launch:
            host = np.concatenate([plan[k] for k in ("N0", "lo0", "K0", "lo1", "chunk_off", "out_off")])
            desc = torch.from_numpy(host).pin_memory().to(rs.device, non_blocking=True)
            _lib.check(_lib.lib().seist_resample_stream(
                self.held[0].data_ptr(), rs.held_bound, chunk.data_ptr(), chunk.numel(), desc.data_ptr(), S, C, int(m.max()),
                rs.taps().data_ptr(), rs.up, rs.down, out.data_ptr(), out.numel(), self.held[1].data_ptr(), _s()), "seist_resample_stream")
            self.held.reverse()
        self.N, self.K = plan["N1"], plan["K1"]
        if self._as_list:
            return [out[C * int(off[s]):C * int(off[s + 1])].view(C, int(m[s])) for s in range(S)]
        return out[:C * int(off[-1])].view(S, C, int(m[0]))
