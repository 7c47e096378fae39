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

A network of mixed input rates takes one Resampler with one rate per station: a list of per-station records in, one
(S, C, T_max) record out, each row NaN past its own output length, and list streams, in one launch per call through a
filter table of the distinct ratios (`filter_table`).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import _lib

MAX_RATIO = 256          # largest up or down after reduction: at most 5 121 taps
_FILL = 16384            # NaNs one CTA writes at most into the tail of a short station's row (a mixed network's record)


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


def stream_plan(N, K, n, up, down, close: bool = False, hl=None) -> dict:
    """One call of a resampling stream, per station, from its inputs received so far N (S,), outputs emitted so far K (S,)
    and this push's lengths n (S,) (ignored at the close).  up, down and the half-length hl (default 10 * max(up, down))
    are ints or per-station arrays (S,).  After N1 inputs output k is final when k < ceil(N1 * up / down)
    and k * down + hl < N1 * up (every input with a nonzero tap has arrived); the close makes every k < ceil(N1 * up / down)
    final.  A station holds the inputs from lo = ceil((K * down - hl) / up) (clipped to [0, N]) on.  Returns int64 arrays
    N0, lo0, K0, lo1, N1, K1 (S,) and the exclusive prefixes chunk_off of the lengths and out_off of K1 - K0 (S + 1,)."""
    if hl is None:
        hl = 10 * np.maximum(up, down)
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


def filter_table(up, down) -> np.ndarray:
    """The filter table of the reduced ratios (up[i], down[i]): (F, 8) int32 rows up, down, hl, nt, tap_off, tile,
    identity, smem as the kernel reads them (include/seist_b200.h); an up == down row is the identity (hl = nt = 0)."""
    up, down = np.ascontiguousarray(up, np.int32), np.ascontiguousarray(down, np.int32)
    table = np.zeros((up.size, 8), np.int32)
    _lib.check(_lib.lib().seist_resample_table(up.size, up.ctypes.data, down.ctypes.data, table.ctypes.data), "seist_resample_table")
    return table


class Resampler:
    """Resample float32 records from input_rate to output_rate on `device` (positive ints; each ratio reduced by its gcd
    may have neither term above 256).  `rs(record)` -> (S, C, ceil(T * up / down)), equal to scipy's
    resample_poly(record, up, down, axis=-1) to fp32 accuracy; `open_stream(S)` -> a ResampleStream.

    input_rate may instead be a sequence of one rate per station: a network of mixed rates, every station's ratio reduced
    on its own and all stations served by one launch per call.  Then `rs(pieces)` takes a list of S (C, T_s) records and
    returns one (S, C, T_max) tensor, row s its record resampled (`output_lengths`) then NaN up to T_max = the longest,
    the form `segments=` of every whole-record consumer takes; `open_stream(S, C)` takes and returns lists.  Per station
    the outputs are bit-identical to Resampler(input_rate[s], output_rate) of its record alone; a station at output_rate
    is copied bit for bit with no latency.  up, down and half_len are then per-station arrays and held_bound the largest."""

    def __init__(self, input_rate, output_rate: int, device="cuda"):
        fout = _check_rate(output_rate, "output_rate")
        self.mixed = isinstance(input_rate, (list, tuple, np.ndarray)) and np.ndim(input_rate) == 1
        rates = [_check_rate(r, f"input_rate[{s}]") for s, r in enumerate(input_rate)] if self.mixed else \
            [_check_rate(input_rate, "input_rate")]
        if not rates:
            raise ValueError("input_rate: expected at least one station")
        ups, downs = [], []
        for s, fin in enumerate(rates):
            g = math.gcd(fin, fout)
            ups.append(fout // g)
            downs.append(fin // g)
            if max(ups[-1], downs[-1]) > MAX_RATIO:
                at = f"station {s}: " if self.mixed else ""
                raise ValueError(f"{at}{fin} -> {fout} Hz reduces to up {ups[-1]}, down {downs[-1]}: neither may exceed {MAX_RATIO}")
        dev = torch.device(device)
        if dev.type != "cuda":
            raise ValueError(f"Resampler has no CPU path, got device {dev}")
        if dev.index is None and torch.cuda.is_available():
            dev = torch.device("cuda", torch.cuda.current_device())
        self.device = dev
        self.output_rate = fout
        self._taps = None
        if not self.mixed:
            self.input_rate = rates[0]
            self.up, self.down = ups[0], downs[0]
            self.half_len = 10 * max(self.up, self.down)
            self.held_bound = (2 * self.half_len + self.down) // self.up + 1
            return
        self.input_rate = rates
        # one table row per distinct ratio; station s applies row filt[s]
        ratios = sorted(set(zip(ups, downs)))
        self.filt = np.array([ratios.index(r) for r in zip(ups, downs)], np.int64)
        self.table = filter_table([u for u, _ in ratios], [d for _, d in ratios])
        self.up, self.down = np.array(ups, np.int64), np.array(downs, np.int64)
        self.half_len = self.table[self.filt, 2].astype(np.int64)
        self.tile = self.table[self.filt, 5].astype(np.int64)
        self.held_bound = int(((2 * self.half_len + self.down) // self.up + 1).max())
        self.smem = int(self.table[:, 7].max())
        self._table = None

    @property
    def identity(self) -> bool:
        return self.up == self.down

    def output_lengths(self, T):
        """Output samples of records of T input samples: ceil(T * up / down), per station for a mixed network."""
        return _ceil_div(np.asarray(T, np.int64) * self.up, self.down)

    def taps(self) -> torch.Tensor:
        """The polyphase table on the device, uploaded on first use; for a mixed network every distinct ratio's taps at
        its tap_off, concatenated."""
        if self._taps is None:
            if self.mixed:
                up, down, nt, off = self.table[:, 0], self.table[:, 1], self.table[:, 3], self.table[:, 4]
                host = np.zeros(max(1, int((off + up * nt).max())), np.float32)
                for i in range(len(self.table)):
                    if up[i] != down[i]:
                        host[off[i]:off[i] + up[i] * nt[i]] = polyphase_taps(int(up[i]), int(down[i])).reshape(-1)
                self._table = torch.from_numpy(self.table).to(self.device)
            else:
                host = polyphase_taps(self.up, self.down)
            self._taps = torch.from_numpy(host).to(self.device)
        return self._taps

    def _check(self, t: torch.Tensor, what: str):
        if not torch.is_tensor(t) or t.dtype != torch.float32 or not t.is_cuda or t.device != self.device or not t.is_contiguous():
            got = f"{tuple(t.shape)} {t.dtype} on {t.device}" if torch.is_tensor(t) else type(t).__name__
            raise ValueError(f"{what}: expected a contiguous float32 CUDA tensor on {self.device}, got {got}")

    def __call__(self, record):
        if self.mixed:
            return self._network(record)
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

    def _network(self, pieces) -> torch.Tensor:
        S = len(self.input_rate)
        if torch.is_tensor(pieces) or not isinstance(pieces, (list, tuple)) or len(pieces) != S:
            got = tuple(pieces.shape) if torch.is_tensor(pieces) else type(pieces).__name__
            raise ValueError(f"a network of {S} input rates takes a list of {S} (C, T_s) records, got {got}")
        C = pieces[0].shape[0] if torch.is_tensor(pieces[0]) and pieces[0].dim() == 2 else 0
        for s, x in enumerate(pieces):
            if not torch.is_tensor(x) or x.dim() != 2 or x.shape[0] != C or C < 1 or x.shape[1] < 1:
                raise ValueError(f"station {s}: expected a ({C}, T) record with T >= 1, got {tuple(x.shape) if torch.is_tensor(x) else x!r}")
            self._check(x, f"station {s}")
        T = np.array([x.shape[1] for x in pieces], np.int64)
        T_out = self.output_lengths(T)
        T_max = int(T_out.max())
        # per channel: the output tiles, then tail CTAs of at most _FILL NaNs each
        per = _ceil_div(T_out, self.tile) + _ceil_div(T_max - T_out, _FILL)
        host = np.concatenate([[x.data_ptr() for x in pieces], T, self.filt, _prefix(C * per)]).astype(np.int64)
        taps = self.taps()
        desc = torch.from_numpy(host).pin_memory().to(self.device, non_blocking=True)
        out = torch.empty(S, C, T_max, device=self.device)
        _lib.check(_lib.lib().seist_resample_multi(desc.data_ptr(), S, C, T_max, int(host[-1]), self._table.data_ptr(), len(self.table),
                                                   self.smem, taps.data_ptr(), out.data_ptr(), _s()), "seist_resample_multi")
        return out

    def open_stream(self, n_stations: int, channels: int = 3) -> "ResampleStream":
        if self.mixed and int(n_stations) != len(self.input_rate):
            raise ValueError(f"a network of {len(self.input_rate)} input rates streams {len(self.input_rate)} stations, got {n_stations}")
        return ResampleStream(self, n_stations, channels)


class ResampleStream:
    """A resampled stream of S stations of C channels (`Resampler.open_stream`).  `push(chunks)` takes an (S, C, n) tensor
    or a list of S (C, n_s) tensors (any n_s >= 0) and returns each station's newly final outputs in the same form: an
    (S, C, m) tensor or a list of S (C, m_s) tensors; a tensor push needs every station to have received as many samples.
    `close()` returns the rest, zeros past each station's end as in the
    whole record, in the form of the last push.  Per station, the concatenated outputs are bit-identical to `rs(record)` of
    its record.  Outputs lag the inputs by hl / up input samples (0.2 s at 100 -> 50 Hz).  Held between calls: N and K
    per station on the host and at most held_bound inputs per row in a fixed (S, C, held_bound) device buffer; a push reads
    nothing back from the device.  The stream of a mixed network takes and returns lists only, each station at its own
    ratio and latency, all stations in one launch per push."""

    def __init__(self, rs: Resampler, n_stations: int, channels: int = 3):
        if int(n_stations) < 1 or int(channels) < 1:
            raise ValueError(f"need at least one station and one channel, got {n_stations}, {channels}")
        self.rs = rs
        self.S, self.C = int(n_stations), int(channels)
        self.held = [torch.zeros(self.S, self.C, rs.held_bound, device=rs.device) for _ in range(2)]
        self.N = np.zeros(self.S, np.int64)
        self.K = np.zeros(self.S, np.int64)
        self.closed = False
        self._as_list = rs.mixed
        self._none = torch.zeros(1, device=rs.device)

    def push(self, chunks):
        if self.closed:
            raise RuntimeError("push() after close()")
        if torch.is_tensor(chunks) and self.rs.mixed:
            raise ValueError(f"a network of mixed input rates takes a list of {self.S} (C, n_s) chunks, got a tensor {tuple(chunks.shape)}")
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
        if self.rs.mixed:
            return self._call(self._plan(n), chunk if chunk.numel() else self._none)
        if self.rs.identity:
            self.N += n
            self.K = self.N.copy()
            return [c.clone() for c in parts] if parts is not None else chunks.clone()
        return self._call(stream_plan(self.N, self.K, n, self.rs.up, self.rs.down), chunk if chunk.numel() else self._none)

    def close(self):
        if self.closed:
            raise RuntimeError("close() after close()")
        if self.rs.mixed:
            out = self._call(self._plan(None), self._none)
            self.closed = True
            return out
        plan = stream_plan(self.N, self.K, None, self.rs.up, self.rs.down, close=True)
        if self.rs.identity:
            plan["out_off"][:] = 0
            plan["K1"] = self.K
        out = self._call(plan, self._none, launch=not self.rs.identity)
        self.closed = True
        return out

    def _plan(self, n) -> dict:
        """A mixed network's call: each station's own ratio and half-length (0 at an identity station, which holds
        nothing), then the filter of each station and its CTAs, max(1, ceil(m_s / tile)) per channel."""
        rs = self.rs
        plan = stream_plan(self.N, self.K, n, rs.up, rs.down, close=n is None, hl=rs.half_len)
        per = np.maximum(1, _ceil_div(plan["K1"] - plan["K0"], rs.tile))
        plan["filt"], plan["cta_off"] = rs.filt, _prefix(self.C * per)
        return plan

    def _call(self, plan: dict, chunk: torch.Tensor, launch: bool = True):
        rs, S, C = self.rs, self.S, self.C
        m = plan["K1"] - plan["K0"]
        off = plan["out_off"]
        out = torch.empty(max(1, C * int(off[-1])), device=rs.device)
        if rs.mixed:
            host = np.concatenate([plan[k] for k in ("N0", "lo0", "K0", "lo1", "chunk_off", "out_off", "filt", "cta_off")])
            taps = rs.taps()
            desc = torch.from_numpy(host).pin_memory().to(rs.device, non_blocking=True)
            _lib.check(_lib.lib().seist_resample_multi_stream(
                self.held[0].data_ptr(), rs.held_bound, chunk.data_ptr(), chunk.numel(), desc.data_ptr(), S, C, int(host[-1]),
                rs._table.data_ptr(), len(rs.table), rs.smem, taps.data_ptr(), out.data_ptr(), out.numel(), self.held[1].data_ptr(),
                _s()), "seist_resample_multi_stream")
            self.held.reverse()
        elif launch:
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
