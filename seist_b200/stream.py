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

from typing import List, Tuple

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


class ContinuousAnnotator:
    """`ann = ContinuousAnnotator(model, window=8192, stride=4096, batch=256, norm_mode="std", stack="mean")`

    * `ann.annotate(record)`: record (S, C, T) float32 on the model's device, T >= window -> probs (S, 3, T) float32 [det,
      P, S].  Three launches per batch of windows (window cut, graph replay, stack) on the current stream, no host sync.
    * `ann.pick_phases(probs, ppk_threshold, spk_threshold, min_peak_dist)` -> {"ppk": (index, prob, offsets), "spk": ...}
      with min_peak_dist in samples (> 1); `ann.split(picks["ppk"])` -> a list of (index, prob) per station.
    * `ann.detect_events(probs, det_threshold)` -> (pairs (E, 2), offsets (S + 1,)).
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

    @torch.no_grad()
    def annotate(self, record: torch.Tensor) -> torch.Tensor:
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

    def pick_phases(self, probs: torch.Tensor, ppk_threshold: float | None = None, spk_threshold: float | None = None,
                    min_peak_dist: int | None = None):
        mpd = self.min_peak_dist if min_peak_dist is None else min_peak_dist
        if mpd is None or int(mpd) <= 1:
            raise ValueError(f"min_peak_dist must be > 1 samples, got {mpd}")
        thr = (self.thresholds["ppk"] if ppk_threshold is None else ppk_threshold,
               self.thresholds["spk"] if spk_threshold is None else spk_threshold)
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
