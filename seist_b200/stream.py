"""Phase picking on continuous records on the device (DESIGN §4.15): sliding-window inference, overlap stacking and
whole-record peak picking / event detection.

The reference only ever runs one window (`demo_predict.py:75` keeps `waveform[:, :8192]`); annotating hours of
3-component data with it means a Python loop that slices, normalises, runs the model and copies every window back for
`_detect_peaks` in numpy.  Here a record `(S, C, T)` that already lives on the GPU is cut into windows of `window`
samples at `stride` (plus one window ending at T when the last regular one falls short), each window normalised as
`DataPreprocessor._normalize` (training/preprocess.py:224-242) does, run through the captured eval plan
(`InferenceGraph`), and the window outputs are stacked into one `(S, 3, T)` probability trace per station (mean or max over
the covering windows).  Picks are `_detect_peaks(mph=threshold, mpd=min_peak_dist, topk=None)` (training/postprocess.py:
15-111) of the whole P / S traces and detections every maximal run of det > threshold (obspy `trigger_onset(p, thr, thr)`,
:114-158), both as CSR tensors.  The numpy restatement is `oracle/stream_ref.py`.  There is no CPU path.
"""
from __future__ import annotations

from typing import List, NamedTuple, Tuple

import numpy as np
import torch

from . import _lib
from .infer import InferenceGraph

_MODES = {"": 0, "std": 1, "max": 2}
_STACK = {"mean": 0, "max": 1}


def _s() -> int:
    return torch.cuda.current_stream().cuda_stream


def window_starts(T: int, window: int, stride: int) -> List[int]:
    """Window starts of one station: k * stride for k = 0 .. (T - window) // stride, then T - window if the last of those
    ends before T."""
    if not (1 <= stride <= window <= T):
        raise ValueError(f"need 1 <= stride <= window <= T, got stride {stride}, window {window}, T {T}")
    starts = list(range(0, T - window + 1, stride))
    if starts[-1] + window < T:
        starts.append(T - window)
    return starts


def _check_probs(probs: torch.Tensor) -> torch.Tensor:
    if not probs.is_cuda or probs.dtype != torch.float32 or probs.dim() != 3 or probs.shape[1] != 3:
        raise RuntimeError("expected (S, 3, T) float32 probabilities on a CUDA device (no CPU path)")
    return probs.contiguous()


def _dense(t: torch.Tensor, shape, what: str, device=None):
    """The in-place kernels write through raw pointers: insist on the exact layout instead of copying."""
    ok = t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.dim() == len(shape)
    ok = ok and all(want is None or got == want for got, want in zip(t.shape, shape))
    if not ok or (device is not None and t.device != device):
        dims = ", ".join("*" if v is None else str(v) for v in shape)
        raise ValueError(f"{what}: expected a contiguous float32 CUDA tensor of shape ({dims}){'' if device is None else f' on {device}'}, "
                         f"got {tuple(t.shape)} {t.dtype} on {t.device}")


def window_batch_(x: torch.Tensor, record: torch.Tensor, window: int, stride: int, w0: int, norm_mode: str = "std") -> torch.Tensor:
    """Fill x (B, C, window) in place with the normalised windows w0 .. w0 + B - 1 of record (S, C, T) (window id
    s * K + k, K windows per station); ids past the last window give zero rows."""
    _dense(record, (None, None, None), "record")
    S, C, T = record.shape
    _dense(x, (None, C, window), "window batch", record.device)
    B = x.shape[0]
    _lib.check(_lib.lib().seist_window_batch(record.data_ptr(), S, C, T, window, stride, w0, B, _MODES[norm_mode], x.data_ptr(), _s()),
               "seist_window_batch")
    return x


def stack_batch_(probs: torch.Tensor, y: torch.Tensor, window: int, stride: int, w0: int, stack: str = "mean") -> torch.Tensor:
    """Add (stack="mean") or max (stack="max") the (B, 3, window) outputs of windows w0 .. w0 + B - 1 into probs
    (S, 3, T).  Batches must be issued in window order, starting at w0 = 0."""
    _dense(probs, (None, 3, None), "probs")
    S, _, T = probs.shape
    _dense(y, (None, 3, window), "window outputs", probs.device)
    _lib.check(_lib.lib().seist_stack_batch(y.data_ptr(), S, T, window, stride, w0, y.shape[0], _STACK[stack], probs.data_ptr(), _s()),
               "seist_stack_batch")
    return probs


def stack_finish_(probs: torch.Tensor, window: int, stride: int, stack: str = "mean") -> torch.Tensor:
    """stack="mean": divide every sample by the number of windows covering it."""
    _dense(probs, (None, 3, None), "probs")
    if stack == "mean":
        S, _, T = probs.shape
        _lib.check(_lib.lib().seist_stack_finish(probs.data_ptr(), S, T, window, stride, _s()), "seist_stack_finish")
    return probs


def _offsets(counts: torch.Tensor) -> torch.Tensor:
    off = torch.zeros(counts.numel() + 1, dtype=torch.int64, device=counts.device)
    torch.cumsum(counts, 0, out=off[1:])
    return off


def pick_peaks(probs: torch.Tensor, channels: Tuple[int, ...], thresholds: Tuple[float, ...], min_peak_dist: int):
    """For each channel: `_detect_peaks(probs[s, channel], mph=threshold, mpd=min_peak_dist, topk=None)` of every station
    as CSR (index (M,) int64, prob (M,) float32, offsets (S + 1,) int64).  Reads the totals once (one host sync)."""
    probs = _check_probs(probs)
    if int(min_peak_dist) <= 1:
        raise ValueError(f"min_peak_dist must be > 1 samples, got {min_peak_dist}")
    S, C, T = probs.shape
    lib = _lib.lib()
    nbytes = lib.seist_peaks_work_bytes(S, T)
    if nbytes < 0:
        raise ValueError(f"pick_peaks: unsupported shape {tuple(probs.shape)}")
    staged = []
    for ch, thr in zip(channels, thresholds):
        work = torch.empty(nbytes, dtype=torch.uint8, device=probs.device)
        counts = torch.empty(S, dtype=torch.int64, device=probs.device)
        _lib.check(lib.seist_peaks_long(probs.data_ptr(), S, C, ch, T, float(thr), int(min_peak_dist), work.data_ptr(), nbytes,
                                        counts.data_ptr(), _s()), "seist_peaks_long")
        staged.append((work, _offsets(counts)))
    totals = torch.stack([off[-1] for _, off in staged]).tolist()
    out = []
    for (work, off), m in zip(staged, totals):
        index = torch.empty(m, dtype=torch.int64, device=probs.device)
        value = torch.empty(m, dtype=torch.float32, device=probs.device)
        if m:
            _lib.check(lib.seist_peaks_long_fill(S, T, work.data_ptr(), nbytes, off.data_ptr(), index.data_ptr(), value.data_ptr(), _s()),
                       "seist_peaks_long_fill")
        out.append((index, value, off))
    return out


def detect_runs(probs: torch.Tensor, channel: int, threshold: float):
    """Every maximal run of probs[s, channel] > threshold as inclusive [on, off], in time order: (pairs (E, 2) int64,
    offsets (S + 1,) int64).  Reads the total once (one host sync)."""
    probs = _check_probs(probs)
    S, C, T = probs.shape
    lib = _lib.lib()
    nbytes = lib.seist_runs_work_bytes(S, T)
    work = torch.empty(nbytes, dtype=torch.uint8, device=probs.device)
    counts = torch.empty(S, dtype=torch.int64, device=probs.device)
    _lib.check(lib.seist_runs_long(probs.data_ptr(), S, C, channel, T, float(threshold), work.data_ptr(), nbytes, counts.data_ptr(), _s()),
               "seist_runs_long")
    off = _offsets(counts)
    pairs = torch.empty(int(off[-1]), 2, dtype=torch.int64, device=probs.device)
    if pairs.numel():
        _lib.check(lib.seist_runs_long_fill(probs.data_ptr(), S, C, channel, T, float(threshold), work.data_ptr(), nbytes, off.data_ptr(),
                                            pairs.data_ptr(), _s()), "seist_runs_long_fill")
    return pairs, off


# ---- streamed records (DESIGN §4.16) ---------------------------------------------------------------------------------
_I64_MAX = (1 << 63) - 1
_I32_MAX = (1 << 31) - 1


def stream_step(S: int, C: int, window: int, stride: int, f0: int, r0: int, f1: int, r1: int, k0: int, nk: int, tail: int = -1,
                kr: int = -1, norm_mode: str = "std", stack: str = "mean") -> _lib.SeistStreamStep:
    """One call of a stream as global sample counts (include/seist_b200.h, SeistStreamStep): R goes r0 -> r1, the final
    prefix f0 -> f1; the call runs regular windows k0 .. k0 + nk - 1 of every station and, at the close, the tail window
    starting at `tail` (-1: none) of a record with kr regular windows."""
    return _lib.SeistStreamStep(f0=f0, r0=r0, f1=f1, r1=r1, k0=k0, tail=tail, kr=kr, S=S, C=C, W=window, P=stride, nk=nk,
                                norm_mode=_MODES[norm_mode], stack_mode=_STACK[stack])


def _ref(step):
    import ctypes
    return ctypes.byref(step)


def stream_window_(x: torch.Tensor, step, tail_raw: torch.Tensor, chunk: torch.Tensor | None, j0: int) -> torch.Tensor:
    """Fill x (B, C, W) with the normalised windows j0 .. j0 + B - 1 of the call `step`, cut from tail_raw (S, C, W) (the
    last min(W, r0) raw samples) followed by chunk (S, C, r1 - r0); ids past the call's last window give zero rows."""
    S, C, W = step.S, step.C, step.W
    _dense(tail_raw, (S, C, W), "kept raw samples")
    _dense(x, (None, C, W), "window batch", tail_raw.device)
    if step.r1 > step.r0:
        _dense(chunk, (S, C, step.r1 - step.r0), "chunk", tail_raw.device)
    _lib.check(_lib.lib().seist_stream_window(_ref(step), tail_raw.data_ptr(), chunk.data_ptr() if step.r1 > step.r0 else None, j0,
                                              x.shape[0], x.data_ptr(), _s()), "seist_stream_window")
    return x


def stream_stack_(acc: torch.Tensor, y: torch.Tensor, step, j0: int, carry: torch.Tensor) -> torch.Tensor:
    """Stack the (B, 3, W) outputs of the call's windows j0 .. j0 + B - 1 into acc (S, 3, r1 - f0); carry (S, 3, W) holds the
    partial sums of [f0, r0) from earlier calls.  Batches in order from j0 = 0."""
    S, W = step.S, step.W
    _dense(carry, (S, 3, W), "carry")
    _dense(acc, (S, 3, step.r1 - step.f0), "partial sums", carry.device)
    _dense(y, (None, 3, W), "window outputs", carry.device)
    _lib.check(_lib.lib().seist_stream_stack(_ref(step), y.data_ptr(), j0, y.shape[0], carry.data_ptr(), acc.data_ptr(), _s()),
               "seist_stream_stack")
    return acc


def stream_emit_(probs: torch.Tensor, carry_out: torch.Tensor, step, carry: torch.Tensor, acc: torch.Tensor) -> torch.Tensor:
    """probs (S, 3, f1 - f0) = the final probabilities of [f0, f1); carry_out (S, 3, W) = the partial sums of [f1, r1)."""
    S, W = step.S, step.W
    _dense(carry, (S, 3, W), "carry")
    _dense(carry_out, (S, 3, W), "carry_out", carry.device)
    _dense(acc, (S, 3, step.r1 - step.f0), "partial sums", carry.device)
    _dense(probs, (S, 3, step.f1 - step.f0), "probs", carry.device)
    if carry_out.data_ptr() == carry.data_ptr():
        raise ValueError("carry_out must not be carry")
    _lib.check(_lib.lib().seist_stream_emit(_ref(step), carry.data_ptr(), acc.data_ptr(), probs.data_ptr(), carry_out.data_ptr(), _s()),
               "seist_stream_emit")
    return probs


def stream_keep_(tail_out: torch.Tensor, step, tail_raw: torch.Tensor, chunk: torch.Tensor | None) -> torch.Tensor:
    """tail_out (S, C, W) = the last min(W, r1) raw samples after the call."""
    S, C, W = step.S, step.C, step.W
    _dense(tail_raw, (S, C, W), "kept raw samples")
    _dense(tail_out, (S, C, W), "tail_out", tail_raw.device)
    if step.r1 > step.r0:
        _dense(chunk, (S, C, step.r1 - step.r0), "chunk", tail_raw.device)
    if tail_out.data_ptr() == tail_raw.data_ptr():
        raise ValueError("tail_out must not be tail_raw")
    _lib.check(_lib.lib().seist_stream_keep(_ref(step), tail_raw.data_ptr(), chunk.data_ptr() if step.r1 > step.r0 else None,
                                            tail_out.data_ptr(), _s()), "seist_stream_keep")
    return tail_out


class StreamOutput(NamedTuple):
    """What one call of a stream made final: probs (S, 3, m) of samples [t0, t0 + m); the picks (index int64 global, prob,
    offsets (S + 1,)) and detection runs (pairs (E, 2) int64 global, offsets) that closed in the call, per station in
    index order."""
    t0: int
    probs: torch.Tensor
    ppk: tuple
    spk: tuple
    det: tuple


class ContinuousStream:
    """A record annotated chunk by chunk (`ContinuousAnnotator.open_stream`).  `push(chunk)` takes (S, C, n) float32 on the
    model's device, any n >= 0; `close()` ends the record.  Each returns a StreamOutput; concatenated, their probs equal
    `annotate(record)` and their picks / runs `pick_phases` / `detect_events` of it (DESIGN §4.16).  Held between calls:
    the last W raw samples, the partial sums of the samples not yet final, and the pending pick clusters and open runs."""

    def __init__(self, ann: "ContinuousAnnotator", n_stations: int):
        self.ann = ann
        self.S, self.C = int(n_stations), ann.in_channels
        self.device = next(ann.model.parameters()).device
        W = ann.window
        self.tail = [torch.zeros(self.S, self.C, W, device=self.device) for _ in range(2)]
        self.carry = [torch.zeros(self.S, 3, W, device=self.device) for _ in range(2)]
        self.R = self.F = self.k = 0
        self.forwards = 0
        self.picker = RaggedPickStream(self.S, self.device, ann.min_peak_dist, ann.thresholds["ppk"], ann.thresholds["spk"],
                                       ann.thresholds["det"])

    @property
    def closed(self) -> bool:
        return self.picker.closed

    @torch.no_grad()
    def push(self, chunk: torch.Tensor) -> StreamOutput:
        if self.closed:
            raise RuntimeError("push() after close()")
        if not chunk.is_cuda:
            raise RuntimeError("ContinuousStream has no CPU path: the chunk must live on the model's CUDA device")
        if chunk.device != self.device:
            raise RuntimeError(f"chunk on {chunk.device}, model on {self.device}")
        if chunk.dtype != torch.float32 or chunk.dim() != 3 or chunk.shape[0] != self.S or chunk.shape[1] != self.C:
            raise ValueError(f"expected a ({self.S}, {self.C}, n) float32 chunk, got {tuple(chunk.shape)} {chunk.dtype}")
        if not chunk.is_contiguous():
            raise ValueError("the chunk must be contiguous")
        W, P = self.ann.window, self.ann.stride
        r1 = self.R + chunk.shape[2]
        k1 = (r1 - W) // P + 1 if r1 >= W else 0
        return self._call(self.R, max(0, r1 - W), r1, k1 - self.k, -1, -1, chunk)

    @torch.no_grad()
    def close(self) -> StreamOutput:
        if self.closed:
            raise RuntimeError("close() after close()")
        W, P, T = self.ann.window, self.ann.stride, self.R
        if T < W:
            raise ValueError(f"the record ({T} samples) is shorter than one window ({W})")
        kr = (T - W) // P + 1
        tail = T - W if (kr - 1) * P + W < T else -1
        return self._call(T, T, T, 0, tail, kr, None)

    def _call(self, r0, f1, r1, nk, tail, kr, chunk):
        ann, S, W = self.ann, self.S, self.ann.window
        step = stream_step(S, self.C, W, ann.stride, self.F, r0, f1, r1, self.k, nk, tail, kr, ann.norm_mode, ann.stack)
        acc = torch.empty(S, 3, r1 - self.F, device=self.device)
        nw = nk + (tail >= 0)
        for j0 in range(0, S * nw, ann.batch):
            stream_window_(ann.graph.x, step, self.tail[0], chunk, j0)
            y = ann.graph.replay()
            stream_stack_(acc, y, step, j0, self.carry[0])
            self.forwards += 1
        probs = torch.empty(S, 3, f1 - self.F, device=self.device)
        stream_emit_(probs, self.carry[1], step, self.carry[0], acc)
        stream_keep_(self.tail[1], step, self.tail[0], chunk)
        self.tail.reverse()
        self.carry.reverse()
        t0 = self.F
        self.R, self.F, self.k = r1, f1, self.k + nk
        ppk, spk, det = self.picker.close(probs) if tail >= 0 or kr >= 0 else self.picker.push(probs)
        return StreamOutput(t0, probs, ppk, spk, det)


# ---- ragged streams: stations that advance at different rates (DESIGN §4.19) -----------------------------------------
_RG_COUNTS = ("f0", "r0", "f1", "r1", "k0", "nk", "tail", "kr")
_RG_OFFS = ("win_off", "chunk_off", "acc_off", "out_off")


def _prefix(counts) -> np.ndarray:
    return np.concatenate([[0], np.cumsum(counts, dtype=np.int64)]).astype(np.int64)


def ragged_plan(R, n, window: int, stride: int, close: bool = False) -> dict:
    """The per-station counts of one call of a ragged stream, from the samples pushed so far R (S,) and this push's
    lengths n (S,) (ignored at the close), by the §4.16 finality rules applied to each station: f0 = max(0, R - W) samples
    are final before the call, k0 = the next regular window; a push runs the regular windows that end by R + n and makes
    max(0, R + n - W) final; the close runs the station's tail window (start T - W, when the last regular window ends
    before T = R) and makes T final.  Returns numpy int64 arrays f0, r0, f1, r1, k0, nk, tail, kr (S,) and the exclusive
    prefix arrays win_off, chunk_off, acc_off, out_off (S + 1,).  Raises ValueError naming the stations with T < W at the
    close."""
    W, P = int(window), int(stride)
    R = np.asarray(R, dtype=np.int64).reshape(-1)
    f0 = np.maximum(R - W, 0)
    k0 = np.where(R >= W, (R - W) // P + 1, 0)
    if close:
        short = np.nonzero(R < W)[0]
        if short.size:
            raise ValueError(f"stations {short.tolist()} hold fewer samples than one window ({W}): "
                             f"{R[short].tolist()}")
        kr = (R - W) // P + 1
        tail = np.where((kr - 1) * P + W < R, R - W, -1)
        r1, f1, nk = R.copy(), R.copy(), np.zeros_like(R)
    else:
        n = np.asarray(n, dtype=np.int64).reshape(-1)
        if n.shape != R.shape or (n < 0).any():
            raise ValueError(f"expected {R.size} non-negative lengths, got {n.tolist()}")
        r1 = R + n
        f1 = np.maximum(r1 - W, 0)
        nk = np.where(r1 >= W, (r1 - W) // P + 1, 0) - k0
        tail = np.full_like(R, -1)
        kr = np.full_like(R, -1)
    plan = dict(f0=f0, r0=R.copy(), f1=f1, r1=r1, k0=k0, nk=nk, tail=tail, kr=kr)
    plan["win_off"] = _prefix(nk + (tail >= 0))
    plan["chunk_off"] = _prefix(r1 - R)
    plan["acc_off"] = _prefix(r1 - f0)
    plan["out_off"] = _prefix(f1 - f0)
    return plan


def ragged_window_ids(plan: dict, stride: int) -> list:
    """The call's packed windows in order as (station, start): each station's regular windows, then its tail window."""
    ids = []
    for s in range(len(plan["f0"])):
        ids += [(s, (int(plan["k0"][s]) + q) * int(stride)) for q in range(int(plan["nk"][s]))]
        if plan["tail"][s] >= 0:
            ids.append((s, int(plan["tail"][s])))
    return ids


def _upload(host: np.ndarray, device) -> torch.Tensor:
    """One small host-to-device copy from pinned memory that does not synchronise the host."""
    return torch.from_numpy(np.ascontiguousarray(host, dtype=np.int64)).pin_memory().to(device, non_blocking=True)


class RaggedStep:
    """One call of a ragged stream: the host plan (`ragged_plan`), its device copy and the SeistRaggedStep pointing into it."""

    def __init__(self, plan: dict, C: int, window: int, stride: int, norm_mode: str = "std", stack: str = "mean", device=None,
                 dev: torch.Tensor | None = None):
        self.plan = plan
        self.S = S = len(plan["f0"])
        self.host = np.concatenate([plan[k] for k in _RG_COUNTS + _RG_OFFS]).astype(np.int64)
        self.dev = _upload(self.host, device) if dev is None else dev
        if self.dev.dtype != torch.int64 or self.dev.numel() < self.host.size or not self.dev.is_cuda:
            raise ValueError("the device copy of a ragged step must be an int64 CUDA tensor holding its plan")
        ptr = [self.dev.data_ptr() + 8 * S * i for i in range(len(_RG_COUNTS))]
        base = self.dev.data_ptr() + 8 * S * len(_RG_COUNTS)
        ptr += [base + 8 * (S + 1) * i for i in range(len(_RG_OFFS))]
        self.n_win = int(plan["win_off"][-1])
        self.max_len = int((plan["r1"] - plan["f0"]).max(initial=0))
        self.desc = _lib.SeistRaggedStep(*ptr, n_win=self.n_win, max_len=self.max_len, S=S, C=int(C), W=int(window), P=int(stride),
                                         norm_mode=_MODES[norm_mode], stack_mode=_STACK[stack])

    def stations(self, j0: int, B: int):
        """The first and last station of windows j0 .. min(j0 + B, n_win) - 1."""
        off = self.plan["win_off"]
        j1 = min(j0 + B, self.n_win) - 1
        return int(np.searchsorted(off, j0, "right") - 1), int(np.searchsorted(off, j1, "right") - 1)


def ragged_stream_step(C: int, window: int, stride: int, R, n, close: bool = False, norm_mode: str = "std", stack: str = "mean",
                       device="cuda") -> RaggedStep:
    """The ragged counterpart of `stream_step`: one call of a ragged stream from the per-station counts R and lengths n."""
    return RaggedStep(ragged_plan(R, n, window, stride, close), C, window, stride, norm_mode, stack, device)


def _flat(t: torch.Tensor, n: int, what: str, device):
    if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.numel() >= max(1, n) and t.device == device):
        raise ValueError(f"{what}: expected a contiguous float32 CUDA tensor on {device} of at least {max(1, n)} elements, "
                         f"got {tuple(t.shape)} {t.dtype} on {t.device}")


def ragged_window_(x: torch.Tensor, step: RaggedStep, tail_raw: torch.Tensor, chunk: torch.Tensor, j0: int) -> torch.Tensor:
    """Fill x (B, C, W) with the normalised windows j0 .. j0 + B - 1 of the call, cut from tail_raw (S, C, W) followed by
    each station's (C, n_s) block of the packed chunk; ids from n_win on give zero rows."""
    d = step.desc
    _dense(tail_raw, (d.S, d.C, d.W), "kept raw samples")
    _dense(x, (None, d.C, d.W), "window batch", tail_raw.device)
    _flat(chunk, d.C * int(step.plan["chunk_off"][-1]), "packed chunk", tail_raw.device)
    _lib.check(_lib.lib().seist_ragged_window(_ref(d), tail_raw.data_ptr(), chunk.data_ptr(), j0, x.shape[0], x.data_ptr(), _s()),
               "seist_ragged_window")
    return x


def ragged_stack_(acc: torch.Tensor, y: torch.Tensor, step: RaggedStep, j0: int, carry: torch.Tensor) -> torch.Tensor:
    """Stack the (B, 3, W) outputs of the call's windows j0 .. j0 + B - 1 into the packed partial sums acc (station s a
    (3, r1 - f0) block at 3 * acc_off[s]); carry (S, 3, W) holds the partial sums of [f0, r0).  Batches in order from 0."""
    d = step.desc
    _dense(carry, (d.S, 3, d.W), "carry")
    _flat(acc, 3 * int(step.plan["acc_off"][-1]), "partial sums", carry.device)
    _dense(y, (None, 3, d.W), "window outputs", carry.device)
    if j0 >= step.n_win:
        return acc
    s0, s1 = step.stations(j0, y.shape[0])
    _lib.check(_lib.lib().seist_ragged_stack(_ref(d), y.data_ptr(), j0, y.shape[0], s0, s1, carry.data_ptr(), acc.data_ptr(), _s()),
               "seist_ragged_stack")
    return acc


def ragged_emit_(probs: torch.Tensor, carry_out: torch.Tensor, step: RaggedStep, carry: torch.Tensor, acc: torch.Tensor) -> torch.Tensor:
    """probs (packed, station s a (3, f1 - f0) block at 3 * out_off[s]) = the final probabilities; carry_out (S, 3, W) =
    the partial sums of [f1, r1)."""
    d = step.desc
    _dense(carry, (d.S, 3, d.W), "carry")
    _dense(carry_out, (d.S, 3, d.W), "carry_out", carry.device)
    _flat(acc, 3 * int(step.plan["acc_off"][-1]), "partial sums", carry.device)
    _flat(probs, 3 * int(step.plan["out_off"][-1]), "probs", carry.device)
    if carry_out.data_ptr() == carry.data_ptr():
        raise ValueError("carry_out must not be carry")
    _lib.check(_lib.lib().seist_ragged_emit(_ref(d), carry.data_ptr(), acc.data_ptr(), probs.data_ptr(), carry_out.data_ptr(), _s()),
               "seist_ragged_emit")
    return probs


def ragged_keep_(tail_out: torch.Tensor, step: RaggedStep, tail_raw: torch.Tensor, chunk: torch.Tensor) -> torch.Tensor:
    """tail_out (S, C, W) = the last min(W, r1[s]) raw samples of each station after the call."""
    d = step.desc
    _dense(tail_raw, (d.S, d.C, d.W), "kept raw samples")
    _dense(tail_out, (d.S, d.C, d.W), "tail_out", tail_raw.device)
    _flat(chunk, d.C * int(step.plan["chunk_off"][-1]), "packed chunk", tail_raw.device)
    if tail_out.data_ptr() == tail_raw.data_ptr():
        raise ValueError("tail_out must not be tail_raw")
    _lib.check(_lib.lib().seist_ragged_keep(_ref(d), tail_raw.data_ptr(), chunk.data_ptr(), tail_out.data_ptr(), _s()),
               "seist_ragged_keep")
    return tail_out


class RaggedStreamOutput(NamedTuple):
    """What one call of a ragged stream made final: per station s, probs[s] (3, m_s) of samples [t0[s], t0[s] + m_s)
    (views into one buffer); the picks and detection runs that closed, as StreamOutput's CSR tuples."""
    t0: list
    probs: list
    ppk: tuple
    spk: tuple
    det: tuple


class RaggedPickStream:
    """The probability side of a stream: takes the final probabilities of S rows in order, stretch after stretch, and
    returns the picks and detection runs that closed (DESIGN §4.16, §4.19).  `push(probs)` takes one (S, 3, m) float32
    tensor (every row a stretch of m samples) or S (3, m_s) float32 tensors, any m, m_s >= 0; each row keeps its own final
    count F_s.  A candidate is decided once the sample after it is final; a cluster of candidates (consecutive gaps <=
    min_peak_dist) is resolved once its last candidate c has c + min_peak_dist <= F_s - 2, so a pick waits for its cluster
    to close.  A run closes once the sample after its end is final.  `t0` (an int or one per row) is the global index of
    each row's first sample."""

    def __init__(self, n_stations: int, device, min_peak_dist: int, ppk_threshold: float = 0.3, spk_threshold: float = 0.3,
                 det_threshold: float = 0.5, t0=0):
        if min_peak_dist is None or int(min_peak_dist) <= 1:
            raise ValueError(f"min_peak_dist must be > 1 samples, got {min_peak_dist}")
        if int(n_stations) < 1:
            raise ValueError(f"need at least one station, got {n_stations}")
        self.S, self.device, self.mpd = int(n_stations), torch.device(device), int(min_peak_dist)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.thr = (float(det_threshold), float(ppk_threshold), float(spk_threshold))
        self.t0 = np.broadcast_to(np.asarray(t0, dtype=np.int64), (self.S,)).copy()
        self.F = self.t0.copy()
        self.closed = False
        self.look = torch.full((self.S, 3, 2), float("-inf"), device=self.device)
        self.open = torch.full((self.S,), -1, dtype=torch.int64, device=self.device)
        self.pend = {1: None, 2: None}        # per pick channel: (work, capc, max_L, base (S,)) of the previous call
        self.max_pend = {1: 0, 2: 0}
        self.first_pend = {1: np.full(self.S, _I64_MAX, np.int64), 2: np.full(self.S, _I64_MAX, np.int64)}
        self._none = torch.zeros(1, device=self.device)

    def push(self, probs):
        """The next final stretch of every row (one (S, 3, m) tensor or a sequence of S (3, m_s) tensors) -> (ppk, spk, det)
        that closed."""
        return self._stretches(probs, False)

    def close(self, probs=None):
        """The last stretches: every pending cluster and open run closes; each row's sample F_s - 1 ends its record."""
        if probs is None:
            probs = [torch.empty(3, 0, device=self.device) for _ in range(self.S)]
        return self._stretches(probs, True)

    def _stretches(self, probs, last: bool):
        if self.closed:
            raise RuntimeError("the stream is closed")
        dense = torch.is_tensor(probs)             # one stretch of m samples per row, already packed
        if dense:
            _dense(probs, (self.S, 3, None), "probabilities", self.device)
            m = np.full(self.S, probs.shape[2], np.int64)
        else:
            if len(probs) != self.S:
                raise ValueError(f"expected {self.S} stretches, got {len(probs)}")
            for p in probs:
                if not p.is_cuda:
                    raise RuntimeError("RaggedPickStream has no CPU path: the probabilities must live on a CUDA device")
                _dense(p, (3, None), "probabilities", self.device)
            m = np.array([p.shape[1] for p in probs], dtype=np.int64)
        host, meta = self._plan(m, last)
        if not m.any():
            flat = self._none
        else:
            flat = probs.view(-1) if dense else torch.cat([p.reshape(-1) for p in probs])
        return self._run(flat, m, last, host, _upload(host, self.device), meta)

    def _plan(self, m: np.ndarray, last: bool):
        """The per-row descriptor of one call on the host (raises before any launch) and its host-side sizes."""
        S = self.S
        f0, f1 = self.F, self.F + m
        # `last`: one bool for every row, or a per-row bool array (a gapped stream closes some rows only, DESIGN §4.22)
        last = last if isinstance(last, (bool, np.bool_)) else np.asarray(last, dtype=bool).reshape(S)
        short = np.nonzero(np.logical_and(last, f1 - self.t0 < 3))[0]
        if short.size:
            raise ValueError(f"rows {short.tolist()} are too short to pick ({(f1 - self.t0)[short].tolist()} samples)")
        L = m + 2 + np.asarray(last, dtype=np.int64)
        max_L = int(L.max())
        if max_L > _I32_MAX:
            raise ValueError(f"a stretch of {int(m.max())} samples is too long for one call")
        g0 = f0 - 2
        lo = np.maximum(1, 3 - (f0 - self.t0))
        hi = m.copy()
        rlo = np.full(S, 2, np.int64)
        rhi = m + 1 + np.asarray(last, dtype=np.int64)
        parts = [_prefix(m), _prefix(L), lo, hi, rlo, rhi, g0]
        meta = {"max_L": max_L, "f1": f1, "span": int(max(0, (hi - lo + 1).max())), "rspan": int((rhi - rlo + 1).max()), "ch": {}}
        for ch in (1, 2):
            base = np.minimum(g0, self.first_pend[ch])
            if (f1 - base >= _I32_MAX - 2).any():
                raise RuntimeError(f"a cluster of candidates spans more than 2^31 samples (channel {ch})")
            lim = np.where(last, _I64_MAX >> 1, f1 - 2 - base).astype(np.int64)
            prev = self.pend[ch]
            delta = base - prev[3] if prev else np.zeros(S, np.int64)
            parts += [lim, base, g0 - base, delta]
            meta["ch"][ch] = (base, self.max_pend[ch] + max_L // 2 + 1)
        return np.concatenate(parts).astype(np.int64), meta

    def _run(self, flat: torch.Tensor, m: np.ndarray, last: bool, host: np.ndarray, dev: torch.Tensor, meta: dict):
        staged = self._stage(flat, host, dev, meta)
        return self._collect(staged, staged["totals"].tolist(), last)   # the one host sync

    def _stage(self, flat: torch.Tensor, host: np.ndarray, dev: torch.Tensor, meta: dict) -> dict:
        """Every launch of a call up to the host read: ext, both channels' peaks and the runs.  `totals` is the int64
        device tensor that `_collect` needs on the host."""
        S, lib, d, max_L = self.S, _lib.lib(), self.device, meta["max_L"]
        ptr = dev.data_ptr()
        prob_off, ext_off = ptr, ptr + 8 * (S + 1)
        lo, hi, rlo, rhi, g0 = (ptr + 8 * (2 * (S + 1) + S * i) for i in range(5))
        chp = {ch: [ptr + 8 * (2 * (S + 1) + S * (5 + 4 * k + i)) for i in range(4)] for k, ch in enumerate((1, 2))}
        n_ext = int(host[2 * (S + 1) - 1])
        ext = torch.empty(max(1, 3 * n_ext), device=d)
        look_out = torch.empty(S, 3, 2, device=d)
        _lib.check(lib.seist_ragged_ext(self.look.data_ptr(), flat.data_ptr(), prob_off, ext_off, S, 3, max_L, ext.data_ptr(),
                                        look_out.data_ptr(), _s()), "seist_ragged_ext")
        staged = []
        for ch in (1, 2):
            lim, base, ishift, delta = chp[ch]
            capc = meta["ch"][ch][1]
            prev = self.pend[ch]
            nbytes = lib.seist_stream_peaks_work_bytes(S, capc, max_L)
            work = torch.empty(nbytes, dtype=torch.uint8, device=d)
            counts = torch.empty(S, dtype=torch.int64, device=d)
            info = torch.empty(2 * S, dtype=torch.int64, device=d)
            _lib.check(lib.seist_ragged_peaks(ext.data_ptr(), ext_off, S, 3, ch, max_L, lo, hi, meta["span"], self.thr[ch], self.mpd, lim,
                                              base, ishift, work.data_ptr(), capc, prev[0].data_ptr() if prev else None,
                                              prev[1] if prev else 0, prev[2] if prev else 0, delta, self.max_pend[ch],
                                              counts.data_ptr(), info.data_ptr(), _s()), "seist_ragged_peaks")
            staged.append((work, capc, _offsets(counts), info))
        rbytes = lib.seist_runs_work_bytes(S, max_L)
        rwork = torch.empty(rbytes, dtype=torch.uint8, device=d)
        rcounts = torch.empty(S, dtype=torch.int64, device=d)
        open_out = torch.empty(S, dtype=torch.int64, device=d)
        _lib.check(lib.seist_ragged_runs(ext.data_ptr(), ext_off, S, 3, 0, max_L, rlo, rhi, meta["rspan"], self.thr[0],
                                         self.open.data_ptr(), open_out.data_ptr(), rwork.data_ptr(), rbytes, rcounts.data_ptr(), _s()),
                   "seist_ragged_runs")
        roff = _offsets(rcounts)
        totals = torch.cat([staged[0][2][-1:], staged[1][2][-1:], roff[-1:], staged[0][3], staged[1][3]])
        return dict(staged=staged, totals=totals, meta=meta, chp=chp, ext=ext, ext_off=ext_off, rlo=rlo, rhi=rhi, g0=g0, rwork=rwork,
                    rbytes=rbytes, roff=roff, open_out=open_out, look_out=look_out)

    def _collect(self, st: dict, tot: list, last: bool):
        """The rest of a call once its totals are on the host: the picks and runs that closed, and the carried state."""
        S, lib, d = self.S, _lib.lib(), self.device
        staged, meta, chp, ext, ext_off = st["staged"], st["meta"], st["chp"], st["ext"], st["ext_off"]
        rlo, rhi, g0, rwork, rbytes, roff, open_out = st["rlo"], st["rhi"], st["g0"], st["rwork"], st["rbytes"], st["roff"], st["open_out"]
        max_L = meta["max_L"]
        out = []
        for i, (ch, (work, capc, off, info)) in enumerate(zip((1, 2), staged)):
            n = tot[i]
            index = torch.empty(n, dtype=torch.int64, device=d)
            value = torch.empty(n, dtype=torch.float32, device=d)
            if n:
                _lib.check(lib.seist_ragged_peaks_fill(S, max_L, work.data_ptr(), capc, chp[ch][1], off.data_ptr(), index.data_ptr(),
                                                       value.data_ptr(), _s()), "seist_ragged_peaks_fill")
            out.append((index, value, off))
            o = 3 + 2 * S * i
            self.max_pend[ch] = max(tot[o:o + S])
            self.first_pend[ch] = np.array(tot[o + S:o + 2 * S], dtype=np.int64)
            self.pend[ch] = (work, capc, max_L, meta["ch"][ch][0])
        pairs = torch.empty(tot[2], 2, dtype=torch.int64, device=d)
        _lib.check(lib.seist_ragged_runs_fill(ext.data_ptr(), ext_off, S, 3, 0, max_L, rlo, rhi, meta["rspan"], self.thr[0], g0,
                                              self.open.data_ptr(), open_out.data_ptr(), rwork.data_ptr(), rbytes, roff.data_ptr(),
                                              pairs.data_ptr() if pairs.numel() else None, _s()), "seist_ragged_runs_fill")
        self.open = open_out
        self.look = st["look_out"]
        self.F = meta["f1"]
        self.closed = last
        return out[0], out[1], (pairs, roff)


class RaggedStream:
    """A record whose stations advance at different rates (`ContinuousAnnotator.open_ragged_stream`).  `push(chunks)` takes
    S float32 tensors (C, n_s) on the model's device, any n_s >= 0 (0: no new data from that station); `close()` ends every
    station's record at its own length.  Each station follows the §4.16 finality rules on its own counts, with sample
    indices counted from its own first sample; the windows of all stations in a call share the batched forward.  Each
    call returns a RaggedStreamOutput; per station, concatenated, its probs equal `annotate` of that station's record and
    its picks / runs `pick_phases` / `detect_events` of it (DESIGN §4.19)."""

    def __init__(self, ann: "ContinuousAnnotator", n_stations: int):
        if int(n_stations) < 1:
            raise ValueError(f"need at least one station, got {n_stations}")
        self.ann = ann
        self.S, self.C = int(n_stations), ann.in_channels
        self.device = next(ann.model.parameters()).device
        W = ann.window
        self.tail = [torch.zeros(self.S, self.C, W, device=self.device) for _ in range(2)]
        self.carry = [torch.zeros(self.S, 3, W, device=self.device) for _ in range(2)]
        self.R = np.zeros(self.S, np.int64)
        self.forwards = 0
        self.picker = RaggedPickStream(self.S, self.device, ann.min_peak_dist, ann.thresholds["ppk"], ann.thresholds["spk"],
                                       ann.thresholds["det"])
        self._none = torch.zeros(1, device=self.device)

    @property
    def closed(self) -> bool:
        return self.picker.closed

    @torch.no_grad()
    def push(self, chunks) -> RaggedStreamOutput:
        return self._call(*self._prepare(chunks), False)

    def _prepare(self, chunks):
        """Validate a push (raises before any launch) -> (the call's plan, the chunks packed at C * chunk_off[s])."""
        if self.closed:
            raise RuntimeError("push() after close()")
        if len(chunks) != self.S:
            raise ValueError(f"expected {self.S} chunks (one per station), got {len(chunks)}")
        for s, c in enumerate(chunks):
            if not torch.is_tensor(c) or not c.is_cuda:
                raise RuntimeError(f"station {s}: RaggedStream has no CPU path, the chunk must live on the model's CUDA device")
            if c.device != self.device:
                raise RuntimeError(f"station {s}: chunk on {c.device}, model on {self.device}")
            if c.dtype != torch.float32 or c.dim() != 2 or c.shape[0] != self.C:
                raise ValueError(f"station {s}: expected a ({self.C}, n) float32 chunk, got {tuple(c.shape)} {c.dtype}")
            if not c.is_contiguous():
                raise ValueError(f"station {s}: the chunk must be contiguous")
        plan = ragged_plan(self.R, [c.shape[1] for c in chunks], self.ann.window, self.ann.stride)
        chunk = torch.cat([c.reshape(-1) for c in chunks]) if plan["chunk_off"][-1] else self._none
        return plan, chunk

    @torch.no_grad()
    def close(self) -> RaggedStreamOutput:
        if self.closed:
            raise RuntimeError("close() after close()")
        return self._call(ragged_plan(self.R, None, self.ann.window, self.ann.stride, close=True), self._none, True)

    def _call(self, plan: dict, chunk: torch.Tensor, last: bool) -> RaggedStreamOutput:
        ann, W = self.ann, self.ann.window
        m = plan["f1"] - plan["f0"]
        pick_host, meta = self.picker._plan(m, last)
        nstep = len(_RG_COUNTS) * self.S + len(_RG_OFFS) * (self.S + 1)
        host = np.concatenate([np.concatenate([plan[k] for k in _RG_COUNTS + _RG_OFFS]), pick_host])
        dev = _upload(host, self.device)                             # the call's one descriptor copy
        step = RaggedStep(plan, self.C, W, ann.stride, ann.norm_mode, ann.stack, self.device, dev[:nstep])
        acc = torch.empty(max(1, 3 * int(plan["acc_off"][-1])), device=self.device)
        for j0 in range(0, step.n_win, ann.batch):
            ragged_window_(ann.graph.x, step, self.tail[0], chunk, j0)
            y = ann.graph.replay()
            ragged_stack_(acc, y, step, j0, self.carry[0])
            self.forwards += 1
        out = plan["out_off"]
        probs = torch.empty(max(1, 3 * int(out[-1])), device=self.device)
        ragged_emit_(probs, self.carry[1], step, self.carry[0], acc)
        ragged_keep_(self.tail[1], step, self.tail[0], chunk)
        self.tail.reverse()
        self.carry.reverse()
        self.R = plan["r1"].copy()
        ppk, spk, det = self.picker._run(probs, m, last, pick_host, dev[nstep:], meta)
        views = [probs[3 * int(out[s]):3 * int(out[s + 1])].view(3, int(m[s])) for s in range(self.S)]
        return RaggedStreamOutput(plan["f0"].tolist(), views, ppk, spk, det)


# ---- whole records with data gaps (DESIGN §4.21) ----------------------------------------------------------------------
_SEG_ROWS = 1 << 16          # segment rows read back by the one host synchronisation of gap_segments
_MAX_ROWS = 65535            # rows of one ragged pick call (grid.y)


class Segments(NamedTuple):
    """The gap-free segments of a record (S, C, T) (`gap_segments`): a gap sample is one where any channel is not finite,
    a segment a maximal run of other samples, inclusive [on, off], in station order then time order.  A segment of at
    least `window` samples is annotated.  On the device: pairs (G, 2) int64 [on, off], offsets (S + 1,) int64 (station s
    holds segments offsets[s] .. offsets[s + 1] - 1), annotated (G,) bool and station (G,) int64; on the host the planner's
    copies on, off (G,) and host_offsets (S + 1,) (numpy int64); the (S, T), device and window it was made for."""
    pairs: torch.Tensor
    offsets: torch.Tensor
    annotated: torch.Tensor
    station: torch.Tensor
    on: np.ndarray
    off: np.ndarray
    host_offsets: np.ndarray
    shape: Tuple[int, int]
    device: torch.device
    window: int


def gap_segments(record: torch.Tensor, window: int) -> Segments:
    """The Segments of record (S, C, T) float32 on a CUDA device for windows of `window` samples.  One pass over the
    record counts each station's segments, a second writes their [on, off]; one host synchronisation reads the counts and
    the table (a second one only when the record holds more than 65 536 segments)."""
    if not record.is_cuda:
        raise RuntimeError("gap_segments has no CPU path: the record must live on a CUDA device")
    if record.dtype != torch.float32 or record.dim() != 3:
        raise ValueError(f"expected a (S, C, T) float32 record, got {tuple(record.shape)} {record.dtype}")
    S, C, T = record.shape
    if not (1 <= S <= 65535 and C >= 1 and 1 <= T <= _I32_MAX and int(window) >= 1):
        raise ValueError(f"need 1 <= S <= 65535, C >= 1, 1 <= T < 2^31 and window >= 1, got {tuple(record.shape)}, window {window}")
    record = record.contiguous()
    lib, dev = _lib.lib(), record.device
    nbytes = lib.seist_runs_work_bytes(S, T)
    work = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    counts = torch.empty(S, dtype=torch.int64, device=dev)
    _lib.check(lib.seist_gap_segments(record.data_ptr(), S, C, T, work.data_ptr(), nbytes, counts.data_ptr(), _s()), "seist_gap_segments")
    off = _offsets(counts)
    cap = min(_SEG_ROWS, S * ((T + 1) // 2))
    pairs = torch.empty(cap, 2, dtype=torch.int64, device=dev)
    _lib.check(lib.seist_gap_segments_fill(record.data_ptr(), S, C, T, work.data_ptr(), nbytes, off.data_ptr(), pairs.data_ptr(), cap,
                                           _s()), "seist_gap_segments_fill")
    host = torch.cat([off, pairs.view(-1)]).cpu().numpy()                  # the one host synchronisation
    host_off = host[:S + 1].copy()
    G = int(host_off[-1])
    if G > cap:
        pairs = torch.empty(G, 2, dtype=torch.int64, device=dev)
        _lib.check(lib.seist_gap_segments_fill(record.data_ptr(), S, C, T, work.data_ptr(), nbytes, off.data_ptr(), pairs.data_ptr(), G,
                                               _s()), "seist_gap_segments_fill")
        table = pairs.cpu().numpy().reshape(-1, 2)
    else:
        pairs = pairs[:G]
        table = host[S + 1:S + 1 + 2 * G].reshape(-1, 2)
    on, off_h = table[:, 0].copy(), table[:, 1].copy()
    station = torch.repeat_interleave(torch.arange(S, device=dev), counts, output_size=G)     # G is known: no second sync
    annotated = (pairs[:, 1] - pairs[:, 0] + 1 >= int(window)).contiguous()
    return Segments(pairs, off, annotated, station, on, off_h, host_off, (S, T), dev, int(window))


def check_segments(segs, S: int, T: int, device, window: int | None = None):
    """Raise ValueError (before any launch) unless segs is a Segments made for a record (S, ., T) on `device` (and for
    `window` when given), its device tensors of the right dtype, rank and size.  The contents are not read."""
    if not isinstance(segs, Segments):
        raise ValueError(f"expected Segments (gap_segments / ContinuousAnnotator.segments), got {type(segs).__name__}")
    device = torch.device(device)
    if tuple(segs.shape) != (S, T) or torch.device(segs.device) != device:
        raise ValueError(f"segments made for (S, T) {tuple(segs.shape)} on {segs.device}, the record is ({S}, {T}) on {device}")
    if window is not None and segs.window != window:
        raise ValueError(f"segments made for windows of {segs.window} samples, the annotator's window is {window}")
    G = len(segs.on)
    for t, what, dtype, shape in ((segs.pairs, "pairs", torch.int64, (G, 2)), (segs.offsets, "offsets", torch.int64, (S + 1,)),
                                  (segs.annotated, "annotated", torch.bool, (G,)), (segs.station, "station", torch.int64, (G,))):
        if not (torch.is_tensor(t) and t.is_cuda and t.device == device and t.dtype == dtype and tuple(t.shape) == shape and
                t.is_contiguous()):
            raise ValueError(f"segments.{what}: expected a contiguous {dtype} CUDA tensor of shape {shape} on {device}, "
                             f"got {tuple(t.shape) if torch.is_tensor(t) else type(t).__name__}"
                             f"{f' {t.dtype} on {t.device}' if torch.is_tensor(t) else ''}")
    if len(segs.off) != G or len(segs.host_offsets) != S + 1:
        raise ValueError(f"segments: host copies of {len(segs.off)} segments and {len(segs.host_offsets)} offsets, expected {G} and {S + 1}")


def segment_plan(on, off, window: int, stride: int, batch: int) -> dict:
    """The packing of all segments' windows, `batch` at a time, from the inclusive [on, off] of each segment (G,): K (G,)
    = len(window_starts(off - on + 1, window, stride)) for a segment of at least `window` samples, else 0; win_off
    (G + 1,) its exclusive prefix; first, last (n_batches,) the first and last segment whose windows batch b holds
    (windows b * batch .. min((b + 1) * batch, win_off[G]) - 1).  numpy int64 arrays."""
    W, P, B = int(window), int(stride), int(batch)
    if not (1 <= P <= W and B >= 1):
        raise ValueError(f"need 1 <= stride <= window and batch >= 1, got stride {P}, window {W}, batch {B}")
    on = np.asarray(on, dtype=np.int64).reshape(-1)
    n = np.asarray(off, dtype=np.int64).reshape(-1) - on + 1
    ann = n >= W
    kr = np.where(ann, (n - W) // P + 1, 0)
    K = np.where(ann, kr + ((kr - 1) * P + W < n), 0).astype(np.int64)
    win_off = _prefix(K)
    j0 = np.arange(0, int(win_off[-1]), B, dtype=np.int64)
    j1 = np.minimum(j0 + B, win_off[-1]) - 1
    first = (np.searchsorted(win_off, j0, "right") - 1).astype(np.int64)
    last = (np.searchsorted(win_off, j1, "right") - 1).astype(np.int64)
    return {"K": K, "win_off": win_off, "first": first, "last": last}


def segment_window_(x: torch.Tensor, record: torch.Tensor, segs: Segments, win_off: torch.Tensor, n_win: int, window: int, stride: int,
                    j0: int, norm_mode: str = "std") -> torch.Tensor:
    """Fill x (B, C, window) in place with the normalised packed segment windows j0 .. j0 + B - 1 (win_off (G + 1,) int64
    on the device, `segment_plan`), cut from record (S, C, T) in place; ids from n_win on give zero rows."""
    _dense(record, (None, None, None), "record")
    S, C, T = record.shape
    _dense(x, (None, C, window), "window batch", record.device)
    G = len(segs.on)
    if n_win > 0 and G:
        _lib.check(_lib.lib().seist_segment_window(record.data_ptr(), S, C, T, segs.pairs.data_ptr(), segs.station.data_ptr(),
                                                   win_off.data_ptr(), G, n_win, window, stride, j0, x.shape[0], _MODES[norm_mode],
                                                   x.data_ptr(), _s()), "seist_segment_window")
    return x


def segment_stack_(probs: torch.Tensor, y: torch.Tensor, segs: Segments, win_off: torch.Tensor, n_win: int, window: int, stride: int,
                   j0: int, g0: int, g1: int, stack: str = "mean") -> torch.Tensor:
    """Stack the (B, 3, window) outputs of packed windows j0 .. j0 + B - 1 into probs (S, 3, T) at their segments' samples;
    g0 .. g1 the segments those windows belong to.  Batches in order from j0 = 0."""
    _dense(probs, (None, 3, None), "probs")
    S, _, T = probs.shape
    _dense(y, (None, 3, window), "window outputs", probs.device)
    _lib.check(_lib.lib().seist_segment_stack(y.data_ptr(), S, T, segs.pairs.data_ptr(), segs.station.data_ptr(), win_off.data_ptr(),
                                              len(segs.on), n_win, window, stride, j0, y.shape[0], g0, g1, _STACK[stack],
                                              probs.data_ptr(), _s()), "seist_segment_stack")
    return probs


def segment_finish_(probs: torch.Tensor, segs: Segments, window: int, stride: int, stack: str = "mean") -> torch.Tensor:
    """stack="mean": divide every sample of an annotated segment by its covering windows; NaN outside every annotated
    segment (both modes)."""
    _dense(probs, (None, 3, None), "probs")
    S, _, T = probs.shape
    G = len(segs.on)
    _lib.check(_lib.lib().seist_segment_finish(probs.data_ptr(), S, T, segs.pairs.data_ptr() if G else None, segs.offsets.data_ptr(),
                                               G, window, stride, _STACK[stack], _s()), "seist_segment_finish")
    return probs


def segment_groups(lengths, max_rows: int = _MAX_ROWS) -> list:
    """The picking groups of the annotated segments of lengths (n,): rows whose lengths share a power-of-two class
    [2^k, 2^(k+1)), in row order, at most max_rows per group.  A group's rows are padded to its longest row, so its
    work stays within twice its own samples.  A list of int64 row arrays, longest class first."""
    lengths = np.asarray(lengths, dtype=np.int64).reshape(-1)
    if lengths.size and lengths.min() < 1:
        raise ValueError("segment lengths must be positive")
    cls = np.floor(np.log2(np.maximum(lengths, 1))).astype(np.int64)
    groups = []
    for k in np.unique(cls)[::-1]:
        r = np.nonzero(cls == k)[0].astype(np.int64)
        groups += [r[i:i + max_rows] for i in range(0, r.size, max_rows)]
    return groups


def pick_segments(probs: torch.Tensor, segs: Segments, thr, mpd: int, det_thr: float = 0.5):
    """P and S picks (thr = their thresholds) of every annotated segment as its own record, as two per-station CSR
    (index, prob, offsets) in index order.  The segments are picked as the rows of closing RaggedPickStream calls (row t0
    = on), one per `segment_groups` group, each group's rows packed by one gather launch; all groups are staged before
    one host synchronisation reads their totals, and the picks are put back in station and index order on the device."""
    probs = _check_probs(probs)
    S, _, T = probs.shape
    check_segments(segs, S, T, probs.device)
    if int(mpd) <= 1:
        raise ValueError(f"min_peak_dist must be > 1 samples, got {mpd}")
    dev = probs.device
    length = segs.off - segs.on + 1
    ann = length >= segs.window
    rows = np.nonzero(ann)[0].astype(np.int64)                  # row i: the i-th annotated segment
    m = length[rows]
    if (m < 3).any():
        raise ValueError(f"segments of {int(m.min())} samples are too short to pick")
    if rows.size == 0:
        return [(torch.empty(0, dtype=torch.int64, device=dev), torch.empty(0, device=dev), torch.zeros(S + 1, dtype=torch.int64, device=dev))
                for _ in range(2)]
    first_row = _prefix(ann.astype(np.int64))[segs.host_offsets]    # station s's rows start at first_row[s]
    lib = _lib.lib()
    staged = []
    for r in segment_groups(m):
        n, gm = r.size, m[r]
        picker = RaggedPickStream(n, dev, mpd, thr[0], thr[1], det_thr, t0=segs.on[rows[r]])
        host, meta = picker._plan(gm, True)                    # host[:n + 1]: the rows' packed offsets
        desc = _upload(np.concatenate([rows[r], r, host]), dev)
        flat = torch.empty(max(1, 3 * int(host[n])), device=dev)
        _lib.check(lib.seist_segment_gather(probs.data_ptr(), S, T, segs.pairs.data_ptr(), segs.station.data_ptr(), len(segs.on),
                                            desc.data_ptr(), desc[2 * n:].data_ptr(), n, int(gm.max()), flat.data_ptr(), flat.numel(),
                                            _s()), "seist_segment_gather")
        staged.append((picker, desc[n:2 * n], picker._stage(flat, host, desc[2 * n:], meta)))
    tot = torch.cat([st["totals"] for _, _, st in staged]).tolist()    # the one host synchronisation
    out = []
    o = 0
    picks = []
    first = _upload(first_row, dev)
    for picker, _, st in staged:
        k = st["totals"].numel()
        picks.append(picker._collect(st, tot[o:o + k], True)[:2])
        o += k
    for ch in range(2):
        counts = torch.zeros(rows.size, dtype=torch.int64, device=dev)   # picks per row, rows in station and index order
        for (_, pos, _), p in zip(staged, picks):
            counts.index_copy_(0, pos, p[ch][2][1:] - p[ch][2][:-1])
        row_off = _offsets(counts)
        M = sum(p[ch][0].numel() for p in picks)
        index = torch.empty(M, dtype=torch.int64, device=dev)
        value = torch.empty(M, dtype=torch.float32, device=dev)
        for (_, pos, _), p in zip(staged, picks):
            idx, val, off = p[ch]
            if idx.numel():
                row = torch.repeat_interleave(torch.arange(pos.numel(), device=dev), off[1:] - off[:-1], output_size=idx.numel())
                dest = row_off.index_select(0, pos.index_select(0, row)) + torch.arange(idx.numel(), device=dev) - off.index_select(0, row)
                index.index_copy_(0, dest, idx)
                value.index_copy_(0, dest, val)
        out.append((index, value, row_off.index_select(0, first)))
    return out


# ---- streams with data gaps: the segment scan of a push and the host plan of a call (DESIGN §4.22) --------------------
_GS_ROWS = ("station", "kind", "on", "src", "closes") + _RG_COUNTS
_CONT, _INTERIOR, _TRAILING = 0, 1, 2


def gap_stream_state(n_stations: int) -> dict:
    """The host state of a fresh gapped stream (`gap_stream_plan`): per station R, the samples pushed; seg_on, the first
    sample of its open segment (-1: none); seg_R, that segment's samples so far; done, the samples already final."""
    z = np.zeros(int(n_stations), np.int64)
    return dict(R=z.copy(), seg_on=np.full(int(n_stations), -1, np.int64), seg_R=z.copy(), done=z.copy())


def gap_stream_plan(state: dict, n, pieces, window: int, stride: int, close: bool = False) -> dict:
    """One call of a gapped stream on the host, from the carried `state` (`gap_stream_state`), the push lengths n (S,)
    (ignored at the close) and the segments of each station's pushed block, pieces = (station, on, off) (G,) inclusive
    and in the block's own index, in station then time order.  A row is one station's piece of one segment in this call:
    kind 0 continues the station's open segment, 1 opens and closes in the push, 2 opens and stays open.  A row closes
    (`closes`) when a gap sample follows it in the push, or at the close; a closing segment of fewer than `window`
    samples is no row (its samples come out NaN).  Each row carries ragged_plan's counts f0, r0, f1, r1, k0, nk, tail, kr
    in its segment's own index, with the close decided per row, and `on` (its segment's first sample in the station's
    index) and `src` (its first sample in the station's block).  Rows with windows come first, each group in station
    then time order.  Returns the rows, their win_off, chunk_off, acc_off, out_off (rows + 1,), the stations' output
    t0 and length m (S,), and the state after the call."""
    W, P = int(window), int(stride)
    R, seg_on, seg_R, done = (np.asarray(state[k], dtype=np.int64) for k in ("R", "seg_on", "seg_R", "done"))
    S = R.size
    if close:
        n = np.zeros(S, np.int64)
        st = a = b = np.zeros(0, np.int64)
    else:
        n = np.asarray(n, dtype=np.int64).reshape(-1)
        if n.shape != R.shape or (n < 0).any():
            raise ValueError(f"expected {S} non-negative lengths, got {n.tolist()}")
        st, a, b = (np.asarray(x, dtype=np.int64).reshape(-1) for x in pieces)
    cont = (a == 0) & (seg_on[st] >= 0)
    closes = b < n[st] - 1
    at0 = np.zeros(S, bool)
    at0[st[a == 0]] = True
    # an open segment whose push starts with a gap (or the close) ends with no new sample
    ends = np.nonzero((seg_on >= 0) & (close | ((n > 0) & ~at0)))[0]
    station = np.concatenate([st, ends])
    src = np.concatenate([a, np.zeros(ends.size, np.int64)])
    length = np.concatenate([b - a + 1, np.zeros(ends.size, np.int64)])
    is_cont = np.concatenate([cont, np.ones(ends.size, bool)])
    closes = np.concatenate([closes, np.ones(ends.size, bool)])
    on = np.where(is_cont, seg_on[station], R[station] + src)
    r0 = np.where(is_cont, seg_R[station], 0)
    r1 = r0 + length
    kind = np.where(is_cont, _CONT, np.where(closes, _INTERIOR, _TRAILING))
    # the state after the call: the open row of each station that pushed, else none
    new_on, new_R = seg_on.copy(), seg_R.copy()
    moved = (n > 0) | close
    new_on[moved], new_R[moved] = -1, 0
    op = ~closes
    new_on[station[op]], new_R[station[op]] = on[op], r1[op]
    R1 = R + n
    new_done = np.where(new_on >= 0, new_on + np.maximum(new_R - W, 0), R1)
    keep = op | (r1 >= W)
    station, src, on, closes, kind, r0, r1 = (x[keep] for x in (station, src, on, closes, kind, r0, r1))
    f0 = np.maximum(r0 - W, 0)
    k0 = np.where(r0 >= W, (r0 - W) // P + 1, 0)
    kr_c = np.where(r1 >= W, (r1 - W) // P + 1, 0)
    kr = np.where(closes, kr_c, -1)
    tail = np.where(closes & ((kr_c - 1) * P + W < r1), r1 - W, -1)
    f1 = np.where(closes, r1, np.maximum(r1 - W, 0))
    nk = kr_c - k0
    nw = nk + (tail >= 0)
    order = np.lexsort((on, station, nw == 0))
    rows = {k: v[order] for k, v in zip(_GS_ROWS, (station, kind, on, src, closes, f0, r0, f1, r1, k0, nk, tail, kr))}
    plan = dict(rows)
    plan["win_off"] = _prefix(nw[order])
    plan["chunk_off"] = _prefix(rows["r1"] - rows["r0"])
    plan["acc_off"] = _prefix(rows["r1"] - rows["f0"])
    plan["out_off"] = _prefix(rows["f1"] - rows["f0"])
    plan["t0"], plan["m"] = done.copy(), new_done - done
    plan["state"] = dict(R=R1, seg_on=new_on, seg_R=new_R, done=new_done)
    return plan


def gap_stream_segments(chunk: torch.Tensor, chunk_off, channels: int):
    """The segments of each station's block of a packed push: station s's samples are a (C, n_s) block at C *
    chunk_off[s] of chunk (float32 on a CUDA device), chunk_off (S + 1,) on the host.  Returns (station, on, off) (G,)
    numpy int64, inclusive and in each block's own index, in station then time order: the `pieces` of
    `gap_stream_plan`.  One host synchronisation reads the counts and a table of at most 65 536 rows (a second one only
    when the push holds more segments)."""
    if not chunk.is_cuda:
        raise RuntimeError("gap_stream_segments has no CPU path: the chunk must live on a CUDA device")
    chunk_off = np.asarray(chunk_off, dtype=np.int64).reshape(-1)
    S, C = chunk_off.size - 1, int(channels)
    n = np.diff(chunk_off)
    if chunk.dtype != torch.float32 or not chunk.is_contiguous() or S < 1 or S > 65535 or C < 1 or (n < 0).any() or \
            C * int(chunk_off[-1]) > chunk.numel() or n.max(initial=0) > _I32_MAX:
        raise ValueError(f"expected a contiguous float32 chunk holding {S} blocks (C, n_s) at C * chunk_off, 1 <= S <= 65535, "
                         f"0 <= n_s < 2^31, got {tuple(chunk.shape)} {chunk.dtype} and lengths {n.tolist()}")
    z = np.zeros(0, np.int64)
    if chunk_off[-1] == 0:
        return z, z, z
    lib, dev = _lib.lib(), chunk.device
    max_n = int(n.max())
    offs = _upload(chunk_off, dev)
    nbytes = lib.seist_runs_work_bytes(S, max_n)
    work = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    counts = torch.empty(S, dtype=torch.int64, device=dev)
    _lib.check(lib.seist_gap_stream_scan(chunk.data_ptr(), chunk.numel(), offs.data_ptr(), S, C, max_n, work.data_ptr(), nbytes,
                                         counts.data_ptr(), _s()), "seist_gap_stream_scan")
    off = _offsets(counts)
    cap = int(min(_SEG_ROWS, ((n + 1) // 2).sum()))
    pairs = torch.empty(max(cap, 1), 2, dtype=torch.int64, device=dev)
    _lib.check(lib.seist_gap_stream_fill(chunk.data_ptr(), chunk.numel(), offs.data_ptr(), S, C, max_n, work.data_ptr(), nbytes,
                                         off.data_ptr(), pairs.data_ptr(), cap, _s()), "seist_gap_stream_fill")
    host = torch.cat([off, pairs.view(-1)]).cpu().numpy()                  # the one host synchronisation
    host_off = host[:S + 1]
    G = int(host_off[-1])
    if G > cap:
        pairs = torch.empty(G, 2, dtype=torch.int64, device=dev)
        _lib.check(lib.seist_gap_stream_fill(chunk.data_ptr(), chunk.numel(), offs.data_ptr(), S, C, max_n, work.data_ptr(), nbytes,
                                             off.data_ptr(), pairs.data_ptr(), G, _s()), "seist_gap_stream_fill")
        table = pairs.cpu().numpy().reshape(-1, 2)
    else:
        table = host[S + 1:S + 1 + 2 * G].reshape(-1, 2)
    station = np.repeat(np.arange(S, dtype=np.int64), np.diff(host_off))
    return station, table[:, 0].copy(), table[:, 1].copy()


def _reorder(parts, n_pos: int, first: np.ndarray, dev):
    """CSR parts [(pos (n,) device int64, values (tuple of (M, ...) tensors), offsets (n + 1,))], row i of a part going to
    position pos[i] of n_pos -> ((values..., offsets at `first` (S + 1,)), the offsets of every position (n_pos + 1,))
    with every row's entries at its position, in order."""
    counts = torch.zeros(n_pos, dtype=torch.int64, device=dev)
    for pos, _, off in parts:
        counts.index_copy_(0, pos, off[1:] - off[:-1])
    row_off = _offsets(counts)
    out = []
    for v in range(len(parts[0][1])):
        M = sum(p[1][v].shape[0] for p in parts)
        t = parts[0][1][v]
        dst = torch.empty((M,) + tuple(t.shape[1:]), dtype=t.dtype, device=dev)
        for pos, vals, off in parts:
            x = vals[v]
            if x.shape[0]:
                row = torch.repeat_interleave(torch.arange(pos.numel(), device=dev), off[1:] - off[:-1], output_size=x.shape[0])
                dest = row_off.index_select(0, pos.index_select(0, row)) + torch.arange(x.shape[0], device=dev) - off.index_select(0, row)
                dst.index_copy_(0, dest, x)
        out.append(dst)
    return (*out, row_off.index_select(0, _upload(first, dev))), row_off


def gap_pick_positions(plan: dict, flip) -> dict:
    """Where the picks of one gapped-stream call go, from its `gap_stream_plan` and each station's open-row flip before
    the call (GapStream: station s's open segment is picked on row 2s + flip[s]).  Station s owns positions first[s] ..
    first[s + 1] - 1: its open segment's picker row, its k_s interior segments in time order, then the picker row of the
    segment after them.  Returns rows_p (rows,): each row's persistent picker row (the open one for interior rows);
    pos_p (2S,): each persistent picker row's position; inter: the interior rows and pos_i their positions; n_pos and
    first (S + 1,); and the position table station, on, end (n_pos,) int64: the segment [on, end] (station index,
    inclusive) whose picks land at each position.  end is on + r1 - 1 for a row that closes and R - 1 after the call
    for one that stays open; a position without a row in the call emits no pick and gets [0, -1] (DESIGN §4.23)."""
    flip = np.asarray(flip, dtype=np.int64).reshape(-1)
    S = flip.size
    st, kind = plan["station"], plan["kind"]
    rows_p = np.where(kind == _TRAILING, 2 * st + 1 - flip[st], 2 * st + flip[st])
    inter = np.nonzero(kind == _INTERIOR)[0]
    k_st = np.bincount(st[inter], minlength=S).astype(np.int64)
    base = 2 * np.arange(S, dtype=np.int64) + _prefix(k_st)[:-1]
    rank = np.arange(inter.size) - np.searchsorted(st[inter], st[inter])     # each interior row's place in its station
    s_p = np.arange(2 * S) // 2
    pos_p = base[s_p] + np.where(np.arange(2 * S) % 2 == flip[s_p], 0, k_st[s_p] + 1)
    pos_i = base[st[inter]] + 1 + rank
    n_pos = 2 * S + inter.size
    row_pos = pos_p[rows_p]
    row_pos[inter] = pos_i
    on, end = np.zeros(n_pos, np.int64), np.full(n_pos, -1, np.int64)
    on[row_pos] = plan["on"]
    end[row_pos] = np.where(plan["closes"], plan["on"] + plan["r1"] - 1, plan["state"]["R"][st] - 1)
    return dict(rows_p=rows_p, pos_p=pos_p, inter=inter, pos_i=pos_i, n_pos=n_pos, first=np.append(base, n_pos),
                station=np.repeat(np.arange(S, dtype=np.int64), k_st + 2), on=on, end=end)


def _copy_rows(src: torch.Tensor, dst: torch.Tensor, m: np.ndarray, src_base, src_ld, dst_base, dst_ld, dev):
    """seist_gap_stream_copy of the rows with m > 0: (3, m) blocks from src to dst."""
    sel = np.nonzero(m > 0)[0]
    if sel.size == 0:
        return dst
    m_off = _prefix(m[sel])
    t = _upload(np.concatenate([m_off] + [np.asarray(x, dtype=np.int64)[sel] for x in (src_base, src_ld, dst_base, dst_ld)]), dev)
    k = sel.size
    ptr = [t.data_ptr() + 8 * ((k + 1) + k * i) for i in range(4)]
    _lib.check(_lib.lib().seist_gap_stream_copy(src.data_ptr(), src.numel(), t.data_ptr(), *ptr, k, 3 * int(m_off[-1]), dst.data_ptr(),
                                                dst.numel(), _s()), "seist_gap_stream_copy")
    return dst


def _check_chunks(chunks, S: int, C: int, device, what: str):
    """Raise (before any launch) unless chunks are S contiguous float32 (C, n_s) tensors on `device`."""
    if len(chunks) != S:
        raise ValueError(f"expected {S} chunks (one per station), got {len(chunks)}")
    for s, c in enumerate(chunks):
        if not torch.is_tensor(c) or not c.is_cuda:
            raise RuntimeError(f"station {s}: {what} has no CPU path, the chunk must live on the model's CUDA device")
        if c.device != device:
            raise RuntimeError(f"station {s}: chunk on {c.device}, model on {device}")
        if c.dtype != torch.float32 or c.dim() != 2 or c.shape[0] != C:
            raise ValueError(f"station {s}: expected a ({C}, n) float32 chunk, got {tuple(c.shape)} {c.dtype}")
        if not c.is_contiguous():
            raise ValueError(f"station {s}: the chunk must be contiguous")


class GapStream:
    """A stream whose stations' data have gaps (`ContinuousAnnotator.open_gap_stream`): `push(chunks)` and `close()` take
    what RaggedStream's take and return a RaggedStreamOutput.  A gap sample is one where any channel is not finite, a
    segment a maximal run of other samples; each segment is streamed as a record of its own, closing in the call that
    delivers the gap after it.  Per station, concatenated over the calls, probs equal `annotate(rec[None],
    segments=segments(rec[None]))[0]` of the station's record, the picks `pick_phases` with those segments and the runs
    `detect_events` (DESIGN §4.22).  Held between calls, per station: the kept raw tail (C, W) and carry (3, W) of its
    open segment and two picker rows (its open segment's and the next one's)."""

    def __init__(self, ann: "ContinuousAnnotator", n_stations: int):
        if not 1 <= int(n_stations) <= _MAX_ROWS // 2:
            raise ValueError(f"need 1 to {_MAX_ROWS // 2} stations (two picker rows each), got {n_stations}")
        self.ann = ann
        self.S, self.C = int(n_stations), ann.in_channels
        self.device = next(ann.model.parameters()).device
        W = ann.window
        self.tail = torch.zeros(self.S, self.C, W, device=self.device)
        self.carry = torch.zeros(self.S, 3, W, device=self.device)
        self.state = gap_stream_state(self.S)
        self.flip = np.zeros(self.S, np.int64)          # station s's open segment is picked on row 2s + flip[s]
        self.forwards = 0
        self.closed = False
        thr = ann.thresholds
        self._thr = (ann.min_peak_dist, thr["ppk"], thr["spk"], thr["det"])
        self.picker = RaggedPickStream(2 * self.S, self.device, *self._thr)
        self._none = torch.zeros(1, device=self.device)

    @property
    def R(self) -> np.ndarray:
        return self.state["R"]

    @torch.no_grad()
    def push(self, chunks) -> RaggedStreamOutput:
        return self._call(*self._prepare(chunks))[0]

    def _lengths(self, chunks) -> np.ndarray:
        """Validate a push (raises before any launch) -> its lengths n (S,)."""
        if self.closed:
            raise RuntimeError("push() after close()")
        _check_chunks(chunks, self.S, self.C, self.device, "GapStream")
        n = np.array([c.shape[1] for c in chunks], dtype=np.int64)
        if n.max(initial=0) > _I32_MAX:
            raise ValueError(f"a chunk of {int(n.max())} samples is too long for one push")
        return n

    def _prepare(self, chunks):
        """Validate, pack and scan a push -> (the call's plan, the chunks packed at C * chunk_off[s], chunk_off)."""
        n = self._lengths(chunks)
        chunk_off = _prefix(n)
        chunk = torch.cat([c.reshape(-1) for c in chunks]) if chunk_off[-1] else self._none
        pieces = gap_stream_segments(chunk, chunk_off, self.C)     # the push's first host synchronisation
        return gap_stream_plan(self.state, n, pieces, self.ann.window, self.ann.stride), chunk, chunk_off

    @torch.no_grad()
    def close(self) -> RaggedStreamOutput:
        return self._close()[0]

    def _close(self):
        if self.closed:
            raise RuntimeError("close() after close()")
        plan = gap_stream_plan(self.state, None, None, self.ann.window, self.ann.stride, close=True)
        res = self._call(plan, self._none, np.zeros(self.S + 1, np.int64))
        self.closed = True
        return res

    def _annotate(self, plan: dict, chunk: torch.Tensor, chunk_off: np.ndarray) -> torch.Tensor:
        """Every row through the ragged stream's kernels; returns the rows' final probabilities packed at 3 * out_off and
        writes the station state of every row that stays open."""
        ann, dev, C, W, P, B = self.ann, self.device, self.C, self.ann.window, self.ann.stride, self.ann.batch
        lib = _lib.lib()
        nr = len(plan["station"])
        probs = torch.empty(max(1, 3 * int(plan["out_off"][-1])), device=dev)
        if nr == 0:
            return probs
        host = np.concatenate([plan[k] for k in _RG_COUNTS + _RG_OFFS] + [plan["station"], plan["src"], plan["closes"].astype(np.int64)])
        tab = _upload(host, dev)
        base = tab.data_ptr()
        cnt = [base + 8 * nr * i for i in range(len(_RG_COUNTS))]
        o = base + 8 * nr * len(_RG_COUNTS)
        offp = [o + 8 * (nr + 1) * i for i in range(len(_RG_OFFS))]
        o += 8 * (nr + 1) * len(_RG_OFFS)
        t_station = tab[(o - base) // 8:(o - base) // 8 + nr]
        row_src = o + 8 * nr
        span = plan["r1"] - plan["f0"]

        def view(ra, rb):
            return _lib.SeistRaggedStep(*[p + 8 * ra for p in cnt + offp], n_win=int(plan["win_off"][rb]),
                                        max_len=int(span[ra:rb].max(initial=0)), S=rb - ra, C=C, W=W, P=P,
                                        norm_mode=_MODES[ann.norm_mode], stack_mode=_STACK[ann.stack])

        # each row's own (C, n_r) block of the push, and the open segment's state for the rows that continue one
        n_raw = int(plan["chunk_off"][-1])
        rows_raw = torch.empty(max(1, C * n_raw), device=dev)
        if n_raw:
            offs = _upload(chunk_off, dev)
            _lib.check(lib.seist_gap_stream_pack(chunk.data_ptr(), chunk.numel(), offs.data_ptr(), self.S, C, t_station.data_ptr(), row_src,
                                                 offp[1], nr, C * n_raw, rows_raw.data_ptr(), rows_raw.numel(), _s()), "seist_gap_stream_pack")
        tail_in = self.tail.index_select(0, t_station)
        carry_in = self.carry.index_select(0, t_station)
        tail_out = torch.empty_like(tail_in)
        carry_out = torch.empty_like(carry_in)
        acc = torch.empty(max(1, 3 * int(plan["acc_off"][-1])), device=dev)
        n_win, woff = int(plan["win_off"][-1]), plan["win_off"]
        for j0 in range(0, n_win, B):
            s0 = int(np.searchsorted(woff, j0, "right") - 1)
            s1 = int(np.searchsorted(woff, min(j0 + B, n_win) - 1, "right") - 1)
            d = view(s0, s1 + 1)
            _lib.check(lib.seist_ragged_window(_ref(d), tail_in[s0:].data_ptr(), rows_raw.data_ptr(), j0, B, ann.graph.x.data_ptr(), _s()),
                       "seist_ragged_window")
            y = ann.graph.replay()
            _lib.check(lib.seist_ragged_stack(_ref(d), y.data_ptr(), j0, B, 0, s1 - s0, carry_in[s0:].data_ptr(), acc.data_ptr(), _s()),
                       "seist_ragged_stack")
            self.forwards += 1
        for ra in range(0, nr, _MAX_ROWS):
            d = view(ra, min(nr, ra + _MAX_ROWS))
            _lib.check(lib.seist_ragged_emit(_ref(d), carry_in[ra:].data_ptr(), acc.data_ptr(), probs.data_ptr(), carry_out[ra:].data_ptr(),
                                             _s()), "seist_ragged_emit")
        op = np.nonzero(~plan["closes"])[0]
        if op.size:
            for ra in range(0, nr, _MAX_ROWS // C):
                d = view(ra, min(nr, ra + _MAX_ROWS // C))
                _lib.check(lib.seist_ragged_keep(_ref(d), tail_in[ra:].data_ptr(), rows_raw.data_ptr(), tail_out[ra:].data_ptr(), _s()),
                           "seist_ragged_keep")
            idx = _upload(np.concatenate([op, plan["station"][op]]), dev)
            self.tail.index_copy_(0, idx[op.size:], tail_out.index_select(0, idx[:op.size]))
            self.carry.index_copy_(0, idx[op.size:], carry_out.index_select(0, idx[:op.size]))
        return probs

    def _call(self, plan: dict, chunk: torch.Tensor, chunk_off: np.ndarray):
        """One call -> (its RaggedStreamOutput, where its P picks came from: `gap_pick_positions`' table station, on, end
        (host) and pos_off, the device offsets (n_pos + 1,) of the P picks by position)."""
        S, dev = self.S, self.device
        rp = self._annotate(plan, chunk, chunk_off)
        st, kind, m_row = plan["station"], plan["kind"], plan["f1"] - plan["f0"]
        src_base, out_off = 3 * plan["out_off"][:-1], plan["out_off"]
        # each station's contiguous output: its rows' final samples, NaN elsewhere
        m_st, t0 = plan["m"], plan["t0"]
        st_off = _prefix(m_st)
        out = torch.full((max(1, 3 * int(st_off[-1])),), float("nan"), device=dev)
        _copy_rows(rp, out, m_row, src_base, m_row, 3 * st_off[st] + plan["on"] + plan["f0"] - t0[st], m_st[st], dev)
        # the picker: the open segments' rows of the persistent picker, the interior segments as closing groups
        pk = self.picker
        where = gap_pick_positions(plan, self.flip)
        rows_p = where["rows_p"]
        trailing = kind == _TRAILING
        if trailing.any():
            reset = rows_p[trailing]
            pk.t0[reset] = pk.F[reset] = plan["on"][trailing]
            for ch in (1, 2):
                pk.first_pend[ch][reset] = _I64_MAX
            r = _upload(reset, dev)
            pk.look.index_fill_(0, r, float("-inf"))
            pk.open.index_fill_(0, r, -1)
            self.flip[st[trailing]] ^= 1
        pers = kind != _INTERIOR
        m_p = np.zeros(2 * S, np.int64)
        last_p = np.zeros(2 * S, bool)
        m_p[rows_p[pers]] = m_row[pers]
        last_p[rows_p[pers]] = plan["closes"][pers]
        pflat = torch.empty(max(1, 3 * int(m_p.sum())), device=dev)
        p_off = _prefix(m_p)
        _copy_rows(rp, pflat, m_row[pers], src_base[pers], m_row[pers], 3 * p_off[rows_p[pers]], m_row[pers], dev)
        # _stage and _collect launch kernels that read the call's descriptor through raw pointers: hold each device copy
        # here until its _collect has launched
        host, meta = pk._plan(m_p, last_p)
        desc = _upload(host, dev)
        staged = [(pk, desc, pk._stage(pflat, host, desc, meta))]
        inter = where["inter"]
        groups = []
        for g in segment_groups(m_row[inter]) if inter.size else []:
            rr = inter[g]
            gp = RaggedPickStream(rr.size, dev, *self._thr, t0=plan["on"][rr])
            gh, gm = gp._plan(m_row[rr], True)
            flat = torch.empty(max(1, 3 * int(gh[rr.size])), device=dev)
            _copy_rows(rp, flat, m_row[rr], src_base[rr], m_row[rr], 3 * gh[:rr.size], m_row[rr], dev)
            gd = _upload(gh, dev)
            staged.append((gp, gd, gp._stage(flat, gh, gd, gm)))
            groups.append(where["pos_i"][g])
        tot = torch.cat([s["totals"] for _, _, s in staged]).tolist()        # the call's last host synchronisation
        res, o = [], 0
        for p, _, s in staged:
            k = s["totals"].numel()
            res.append(p._collect(s, tot[o:o + k], False))
            o += k
        # per station: its open segment's row, its interior segments in time order, then the row of the segment after them
        pos = [_upload(x, dev) for x in [where["pos_p"]] + groups]
        n_pos, first = where["n_pos"], where["first"]
        ppk, pos_off = _reorder([(ps, r[0][:2], r[0][2]) for ps, r in zip(pos, res)], n_pos, first, dev)
        spk, _ = _reorder([(ps, r[1][:2], r[1][2]) for ps, r in zip(pos, res)], n_pos, first, dev)
        det, _ = _reorder([(ps, r[2][:1], r[2][1]) for ps, r in zip(pos, res)], n_pos, first, dev)
        self.state = plan["state"]
        views = [out[3 * int(st_off[s]):3 * int(st_off[s + 1])].view(3, int(m_st[s])) for s in range(S)]
        table = {k: where[k] for k in ("station", "on", "end")}
        return RaggedStreamOutput(t0.tolist(), views, ppk, spk, det), dict(table, pos_off=pos_off)


class ContinuousAnnotator:
    """`ann = ContinuousAnnotator(model, window=8192, stride=4096, batch=256, norm_mode="std", stack="mean")`

    * `ann.annotate(record)`: record (S, C, T) float32 on the model's device, T >= window -> probs (S, 3, T) float32 [det,
      P, S].  Three launches per batch of windows (window cut, graph replay, stack) on the current stream, no host sync.
    * `ann.pick_phases(probs, ppk_threshold, spk_threshold, min_peak_dist)` -> {"ppk": (index, prob, offsets), "spk": ...}
      with min_peak_dist in samples (> 1); `ann.split(picks["ppk"])` -> a list of (index, prob) per station.
    * `ann.detect_events(probs, det_threshold)` -> (pairs (E, 2), offsets (S + 1,)).
    * `st = ann.open_stream(n_stations)`: the same, chunk by chunk (`st.push(chunk)`, `st.close()`, ContinuousStream);
      thresholds and min_peak_dist are read here.
    * `st = ann.open_ragged_stream(n_stations)`: the same with stations that advance at different rates
      (`st.push([chunk_s (C, n_s) per station])`, `st.close()`, RaggedStream).
    * Records with data gaps (non-finite samples): `segs = ann.segments(record)`, then `annotate(record, segments=segs)`
      and `pick_phases(probs, segments=segs)` treat every gap-free segment of at least `window` samples as a record of
      its own (NaN elsewhere); `detect_events` needs no segments (DESIGN §4.21).
    * `st = ann.open_gap_stream(n_stations)`: a ragged stream whose data have gaps, each station's segments streamed as
      records of their own (`st.push(chunks)`, `st.close()`, GapStream, DESIGN §4.22).
    Only the seist_*_dpk models (a [det, P, S] probability head) are supported."""

    def __init__(self, model, window: int = 8192, stride: int | None = None, batch: int = 256, norm_mode: str = "std",
                 stack: str = "mean"):
        hp = getattr(model, "hp", None)
        if getattr(hp, "head", None) != "dpk" or getattr(hp, "head_out_channels", None) != 3:
            raise NotImplementedError("ContinuousAnnotator annotates with the seist_*_dpk models ([det, P, S] probabilities) only")
        stride = window // 2 if stride is None else stride
        if not (1 <= int(stride) <= int(window)):
            raise ValueError(f"stride must lie in [1, window], got {stride} for window {window}")
        if norm_mode not in _MODES:
            raise ValueError(f"Supported mode: 'max','std', got '{norm_mode}'")
        if stack not in _STACK:
            raise ValueError(f"stack must be 'mean' or 'max', got '{stack}'")
        if int(batch) < 1:
            raise ValueError(f"batch must be >= 1, got {batch}")
        self.model = model
        self.window, self.stride, self.batch = int(window), int(stride), int(batch)
        self.norm_mode, self.stack = norm_mode, stack
        self.in_channels = hp.in_channels
        self.thresholds = {"ppk": 0.3, "spk": 0.3, "det": 0.5}
        self.min_peak_dist = None
        self.graph = InferenceGraph(model, self.batch, self.window)
        y = self.graph.y
        if tuple(y.shape) != (self.batch, 3, self.window) or not y.is_contiguous():
            raise RuntimeError(f"unexpected eval plan output {tuple(y.shape)}")

    @classmethod
    def from_args(cls, model, args, sampling_rate: int, **kwargs) -> "ContinuousAnnotator":
        """From the reference's command-line names (main.py): in_samples, norm_mode, ppk_threshold, spk_threshold,
        det_threshold and min_peak_dist (seconds, times sampling_rate as in postprocess.py:228)."""
        ann = cls(model, window=args.in_samples, norm_mode=args.norm_mode, **kwargs)
        ann.thresholds = {"ppk": float(args.ppk_threshold), "spk": float(args.spk_threshold), "det": float(args.det_threshold)}
        ann.min_peak_dist = int(args.min_peak_dist * sampling_rate)
        return ann

    def window_count(self, T: int) -> int:
        return len(window_starts(T, self.window, self.stride))

    def segments(self, record: torch.Tensor) -> Segments:
        """The gap-free segments of record (S, C, T) for this annotator's window (`gap_segments`); one host sync."""
        return gap_segments(record, self.window)

    @torch.no_grad()
    def annotate(self, record: torch.Tensor, segments: Segments | None = None) -> torch.Tensor:
        dev = next(self.model.parameters()).device
        if not record.is_cuda:
            raise RuntimeError("ContinuousAnnotator has no CPU path: the record must live on the model's CUDA device")
        if record.device != dev:
            raise RuntimeError(f"record on {record.device}, model on {dev}")
        if record.dtype != torch.float32 or record.dim() != 3:
            raise ValueError(f"expected a (S, C, T) float32 record, got {tuple(record.shape)} {record.dtype}")
        S, C, T = record.shape
        if C != self.in_channels:
            raise ValueError(f"the model takes {self.in_channels} channels, the record has {C}")
        if segments is not None:
            check_segments(segments, S, T, dev, self.window)
            return self._annotate_segments(record.contiguous(), segments)
        if T < self.window:
            raise ValueError(f"the record ({T} samples) is shorter than one window ({self.window})")
        record = record.contiguous()
        n = S * self.window_count(T)
        probs = torch.empty(S, 3, T, dtype=torch.float32, device=dev)
        for w0 in range(0, n, self.batch):
            window_batch_(self.graph.x, record, self.window, self.stride, w0, self.norm_mode)
            y = self.graph.replay()
            stack_batch_(probs, y, self.window, self.stride, w0, self.stack)
        return stack_finish_(probs, self.window, self.stride, self.stack)

    def _annotate_segments(self, record: torch.Tensor, segs: Segments) -> torch.Tensor:
        """Every annotated segment as a record of its own, the windows of all segments packed `batch` at a time; NaN
        outside the annotated segments (DESIGN §4.21)."""
        S, _, T = record.shape
        W, P, B = self.window, self.stride, self.batch
        plan = segment_plan(segs.on, segs.off, W, P, B)
        n_win = int(plan["win_off"][-1])
        probs = torch.empty(S, 3, T, dtype=torch.float32, device=record.device)
        if n_win:
            win_off = _upload(plan["win_off"], record.device)
            for b, j0 in enumerate(range(0, n_win, B)):
                segment_window_(self.graph.x, record, segs, win_off, n_win, W, P, j0, self.norm_mode)
                y = self.graph.replay()
                segment_stack_(probs, y, segs, win_off, n_win, W, P, j0, int(plan["first"][b]), int(plan["last"][b]), self.stack)
        return segment_finish_(probs, segs, W, P, self.stack)

    def open_stream(self, n_stations: int) -> ContinuousStream:
        if self.min_peak_dist is None or int(self.min_peak_dist) <= 1:
            raise ValueError(f"min_peak_dist must be > 1 samples, got {self.min_peak_dist}")
        return ContinuousStream(self, n_stations)

    def open_ragged_stream(self, n_stations: int) -> RaggedStream:
        """A stream whose stations advance at different rates (RaggedStream); thresholds and min_peak_dist are read here."""
        if self.min_peak_dist is None or int(self.min_peak_dist) <= 1:
            raise ValueError(f"min_peak_dist must be > 1 samples, got {self.min_peak_dist}")
        return RaggedStream(self, n_stations)

    def open_gap_stream(self, n_stations: int) -> "GapStream":
        """A ragged stream whose stations' data have gaps (GapStream, at most 32 767 stations); thresholds and
        min_peak_dist are read here."""
        if self.min_peak_dist is None or int(self.min_peak_dist) <= 1:
            raise ValueError(f"min_peak_dist must be > 1 samples, got {self.min_peak_dist}")
        return GapStream(self, n_stations)

    def pick_phases(self, probs: torch.Tensor, ppk_threshold: float | None = None, spk_threshold: float | None = None,
                    min_peak_dist: int | None = None, segments: Segments | None = None):
        mpd = self.min_peak_dist if min_peak_dist is None else min_peak_dist
        if mpd is None or int(mpd) <= 1:
            raise ValueError(f"min_peak_dist must be > 1 samples, got {mpd}")
        thr = (self.thresholds["ppk"] if ppk_threshold is None else ppk_threshold,
               self.thresholds["spk"] if spk_threshold is None else spk_threshold)
        if segments is not None:
            if isinstance(segments, Segments) and segments.window != self.window:
                raise ValueError(f"segments made for windows of {segments.window} samples, the annotator's window is {self.window}")
            ppk, spk = pick_segments(probs, segments, thr, int(mpd), self.thresholds["det"])
            return {"ppk": ppk, "spk": spk}
        ppk, spk = pick_peaks(probs, (1, 2), thr, int(mpd))
        return {"ppk": ppk, "spk": spk}

    def detect_events(self, probs: torch.Tensor, det_threshold: float | None = None):
        return detect_runs(probs, 0, self.thresholds["det"] if det_threshold is None else det_threshold)

    @staticmethod
    def split(csr) -> list:
        """CSR (values..., offsets) -> one tuple of the values' slices per station."""
        *vals, off = csr
        o = off.tolist()
        return [tuple(v[o[i]:o[i + 1]] for v in vals) for i in range(len(o) - 1)]
