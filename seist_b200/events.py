"""Characterise picked events on continuous records (DESIGN §4.17): every P pick of a pick list through the polarity,
magnitude, back-azimuth and distance models.

The reference defines how these models see an event: `DataPreprocessor._cut_window` with 0 <= p_position_ratio <= 1
(training/preprocess.py:172-203) cuts `in_samples` with the first P pick at sample int(in_samples * p_position_ratio),
zero-filling what falls outside the trace, and `_normalize` (:224-242) normalises the window per channel.  Here the P
picks of a whole record, as the CSR `ContinuousAnnotator.pick_phases(...)["ppk"]` returns them, are cut straight into the
static inputs of the models' captured eval plans (`InferenceGraph`) by one kernel launch per batch of events
(`seist_event_windows`, csrc/stream.cu), and the outputs come back aligned index for index with the pick list.  The numpy
restatement of the cut is `oracle/event_ref.py`.  `EventCharacterizer.open_stream` does the same for the P picks of a
record streamed chunk by chunk, in the call that emits them (DESIGN §4.18).  There is no CPU path.
"""
from __future__ import annotations

import ctypes
from typing import NamedTuple

import torch

from . import _lib
from .infer import InferenceGraph
from .stream import _I32_MAX, _MODES, ContinuousAnnotator, StreamOutput, _dense, _s

MAX_MODELS = 4              # destinations of one seist_event_windows launch
MAX_WINDOW = 49152          # a row of the window is staged in shared memory


def anchor(window: int, p_position_ratio: float) -> int:
    """Sample of the window that holds the P pick: the reference's `int(window_size * self.p_position_ratio)`."""
    return int(window * p_position_ratio)


def _check_picks(index: torch.Tensor, offsets: torch.Tensor, S: int, device):
    for t, what, shape in ((index, "pick index", None), (offsets, "pick offsets", S + 1)):
        ok = t.is_cuda and t.dtype == torch.int64 and t.dim() == 1 and t.is_contiguous() and t.device == device
        if not ok or (shape is not None and t.numel() != shape):
            want = "(M,)" if shape is None else f"({shape},)"
            raise ValueError(f"{what}: expected a contiguous int64 CUDA tensor of shape {want} on {device}, "
                             f"got {tuple(t.shape)} {t.dtype} on {t.device}")


def event_windows_(xs, record: torch.Tensor, index: torch.Tensor, offsets: torch.Tensor, e0: int, window: int, anchor: int,
                   norm_mode: str = "std"):
    """Fill every x in xs (1 to 4 tensors (B, C, window)) with the normalised P-anchored windows of events e0 .. e0 + B - 1
    of the pick CSR (index (M,) int64, offsets (S + 1,) int64) on record (S, C, T): the pick at sample `anchor`, zeros
    outside the record.  Events >= M and picks outside [0, T) give zero rows."""
    _dense(record, (None, None, None), "record")
    S, C, T = record.shape
    if not 1 <= len(xs) <= MAX_MODELS:
        raise ValueError(f"1 to {MAX_MODELS} destinations, got {len(xs)}")
    for x in xs:
        _dense(x, (xs[0].shape[0], C, window), "event window batch", record.device)
    _check_picks(index, offsets, S, record.device)
    if not (1 <= window <= MAX_WINDOW and 0 <= anchor <= window and T < 2 ** 31 and e0 >= 0):
        raise ValueError(f"need 1 <= window <= {MAX_WINDOW}, 0 <= anchor <= window, T < 2^31 and e0 >= 0, got window {window}, "
                         f"anchor {anchor}, T {T}, e0 {e0}")
    ptrs = (ctypes.c_void_p * MAX_MODELS)(*[x.data_ptr() for x in xs])
    _lib.check(_lib.lib().seist_event_windows(record.data_ptr(), S, C, T, index.data_ptr(), index.numel(), offsets.data_ptr(), e0,
                                              xs[0].shape[0], window, anchor, _MODES[norm_mode], ptrs, len(xs), _s()),
               "seist_event_windows")
    return xs


class EventCharacterizer:
    """`ch = EventCharacterizer({"pmp": m_pmp, "emg": m_emg, ...}, window=8192, p_position_ratio=0.3, batch=256)`

    * `ch(record, ppk)`: record (S, C, T) float32 on the models' device, ppk the P pick CSR (index (M,) int64, ...,
      offsets (S + 1,) int64), e.g. `ContinuousAnnotator.pick_phases(...)["ppk"]` -> {name: outputs}, row i for pick i:
      (M, classes) softmax probabilities of a classification model, (M,) scaled sigmoid of a regression model.
      `ContinuousAnnotator.split((out[name], offsets))` gives them per station.
    * Per batch of events one window cut writes every model's input, then each model's captured eval plan replays; no
      host synchronisation.
    Takes 1 to 4 non-dpk SeisT models (head "cls" or "reg") of one channel count on one CUDA device.  p_position_ratio
    must lie in [0, 1]; the reference's -1 (a random training cut) has no meaning for a given pick."""

    def __init__(self, models: dict, window: int = 8192, *, p_position_ratio: float, batch: int = 256, norm_mode: str = "std"):
        if not isinstance(models, dict) or not 1 <= len(models) <= MAX_MODELS:
            raise ValueError(f"expected a dict of 1 to {MAX_MODELS} models, got {type(models).__name__} of {len(models)}")
        heads, channels, devices = {}, set(), set()
        for name, m in models.items():
            hp = getattr(m, "hp", None)
            head = getattr(hp, "head", None)
            if head not in ("cls", "reg"):
                raise NotImplementedError(f"model {name!r}: EventCharacterizer runs the classification and regression heads "
                                          f"(pmp, emg, baz, dis); got head {head!r} (use ContinuousAnnotator for dpk)")
            heads[name] = head
            channels.add(hp.in_channels)
            devices.add(next(m.parameters()).device)
        if len(channels) != 1:
            raise ValueError(f"the models take different channel counts: {sorted(channels)}")
        if len(devices) != 1 or next(iter(devices)).type != "cuda":
            raise ValueError(f"the models must live on one CUDA device, got {sorted(map(str, devices))}")
        if not 0 <= float(p_position_ratio) <= 1:
            raise ValueError(f"p_position_ratio must lie in [0, 1], got {p_position_ratio}")
        if not 1 <= int(window) <= MAX_WINDOW:
            raise ValueError(f"window must lie in [1, {MAX_WINDOW}], got {window}")
        if norm_mode not in _MODES:
            raise ValueError(f"Supported mode: 'max','std', got '{norm_mode}'")
        if int(batch) < 1:
            raise ValueError(f"batch must be >= 1, got {batch}")
        self.models, self.heads = dict(models), heads
        self.window, self.batch, self.norm_mode = int(window), int(batch), norm_mode
        self.p_position_ratio = float(p_position_ratio)
        self.anchor = anchor(self.window, p_position_ratio)
        self.in_channels = channels.pop()
        self.device = devices.pop()
        self.graphs = {name: InferenceGraph(m, self.batch, self.window) for name, m in self.models.items()}
        for name, g in self.graphs.items():
            want = 1 if heads[name] == "reg" else self.models[name].hp.head_num_classes
            if tuple(g.y.shape) != (self.batch, want):
                raise RuntimeError(f"model {name!r}: unexpected eval plan output {tuple(g.y.shape)}")

    @classmethod
    def from_args(cls, models: dict, args, **kwargs) -> "EventCharacterizer":
        """From the reference's command-line names (main.py): in_samples, norm_mode and p_position_ratio."""
        return cls(models, window=args.in_samples, p_position_ratio=args.p_position_ratio, norm_mode=args.norm_mode, **kwargs)

    @torch.no_grad()
    def __call__(self, record: torch.Tensor, ppk) -> dict:
        index, offsets = ppk[0], ppk[-1]
        if not record.is_cuda or not index.is_cuda or not offsets.is_cuda:
            raise RuntimeError("EventCharacterizer has no CPU path: the record and the picks must live on the models' CUDA device")
        if record.device != self.device:
            raise RuntimeError(f"record on {record.device}, models on {self.device}")
        if record.dtype != torch.float32 or record.dim() != 3:
            raise ValueError(f"expected a (S, C, T) float32 record, got {tuple(record.shape)} {record.dtype}")
        S, C, T = record.shape
        if C != self.in_channels:
            raise ValueError(f"the models take {self.in_channels} channels, the record has {C}")
        if T >= 2 ** 31:
            raise ValueError(f"record length {T} must stay below 2^31 samples")
        _check_picks(index, offsets, S, self.device)
        return self._run(record.contiguous(), index, offsets)

    def _run(self, record: torch.Tensor, index: torch.Tensor, offsets: torch.Tensor) -> dict:
        M = index.numel()
        out = {name: torch.empty((M,) if self.heads[name] == "reg" else (M, g.y.shape[1]), dtype=torch.float32, device=self.device)
               for name, g in self.graphs.items()}
        xs = [g.x for g in self.graphs.values()]
        for e0 in range(0, M, self.batch):
            event_windows_(xs, record, index, offsets, e0, self.window, self.anchor, self.norm_mode)
            n = min(self.batch, M - e0)
            for name, g in self.graphs.items():
                y = g.replay()
                out[name][e0:e0 + n] = y[:n, 0] if self.heads[name] == "reg" else y[:n]
        return out

    def open_stream(self, annotator: ContinuousAnnotator, n_stations: int) -> "CharacterizedStream":
        """A record picked chunk by chunk by `annotator` (a dpk ContinuousAnnotator, thresholds and min_peak_dist set),
        every P pick characterised in the call that emits it (DESIGN §4.18)."""
        return CharacterizedStream(self, annotator, n_stations)


def stream_history_(out: torch.Tensor, held: torch.Tensor, h0_held: int, chunk: torch.Tensor | None, h0_out: int) -> torch.Tensor:
    """The raw samples [h0_out, h0_held + held.shape[2] + n) of every row, from held (S, C, n_held: samples h0_held ..)
    followed by chunk (S, C, n), written packed into the flat float32 buffer out -> the (S, C, n_out) view of it."""
    _dense(held, (None, None, None), "held samples")
    S, C, n_held = held.shape
    n = 0 if chunk is None else chunk.shape[2]
    if chunk is not None:
        _dense(chunk, (S, C, None), "chunk", held.device)
    _dense(out, (None,), "history buffer", held.device)
    n_out = h0_held + n_held + n - h0_out
    if not (0 <= h0_held <= h0_out and 0 <= n_out <= _I32_MAX and S * C * n_out <= out.numel()):
        raise ValueError(f"need 0 <= h0_held <= h0_out, an output of 0 .. 2^31 - 1 samples and a buffer of S * C * n_out floats, "
                         f"got h0_held {h0_held}, h0_out {h0_out}, n_out {n_out}, buffer {out.numel()}")
    _lib.check(_lib.lib().seist_stream_history(held.data_ptr() if n_held else None, h0_held, n_held, chunk.data_ptr() if n else None, n,
                                               h0_out, S, C, out.data_ptr(), out.numel(), _s()), "seist_stream_history")
    return out[:S * C * n_out].view(S, C, n_out)


class CharacterizedOutput(NamedTuple):
    """One call of a CharacterizedStream: the stream's StreamOutput and {name: outputs} for its P picks, row i for pick i
    of `out.ppk` ((m, classes) probabilities of a classification model, (m,) of a regression model)."""
    out: StreamOutput
    events: dict


class CharacterizedStream:
    """`EventCharacterizer.open_stream(annotator, n_stations)`: `push(chunk (S, C, n))` for any n >= 0, then `close()`, each
    -> CharacterizedOutput.  Concatenated per station, the events equal `ch(record, annotator.pick_phases(
    annotator.annotate(record))["ppk"])` bit for bit, and each comes out in the call that emits its pick (DESIGN §4.18).
    Besides the ContinuousStream's state it holds the raw samples [h0, R) in one of two device buffers: h0 is the retention
    bound max(0, min(first pending P candidate, F - 1) - anchor) of the call before the last non-empty push, below which
    no pick emitted since then starts its window.  `held_samples` = R - h0."""

    def __init__(self, ch: EventCharacterizer, ann: ContinuousAnnotator, n_stations: int):
        dev = next(ann.model.parameters()).device
        if dev != ch.device:
            raise ValueError(f"the annotator's model is on {dev}, the characteriser's models on {ch.device}")
        if ann.in_channels != ch.in_channels:
            raise ValueError(f"the annotator takes {ann.in_channels} channels, the characteriser's models {ch.in_channels}")
        if ch.window - ch.anchor > ann.window:
            raise ValueError(f"the characteriser's window reaches {ch.window - ch.anchor} samples past the pick, more than the "
                             f"annotator's window ({ann.window}): a pick's event window would not be pushed yet when it closes")
        self.ch = ch
        self.stream = ann.open_stream(n_stations)
        self.S, self.C, self.device = self.stream.S, self.stream.C, self.stream.device
        self.buf = [torch.empty(0, device=self.device), torch.empty(0, device=self.device)]
        self.history = self.buf[0].view(self.S, self.C, 0)
        self.h0 = self.R = 0
        self.keep = 0            # the retention bound after the last call

    @property
    def closed(self) -> bool:
        return self.stream.closed

    @property
    def forwards(self) -> int:
        return self.stream.forwards

    @property
    def held_samples(self) -> int:
        return self.R - self.h0

    @torch.no_grad()
    def push(self, chunk: torch.Tensor) -> CharacterizedOutput:
        n = chunk.shape[2] if isinstance(chunk, torch.Tensor) and chunk.dim() == 3 else 0
        if not self.closed and self.R + n - self.keep > _I32_MAX:
            raise ValueError(f"the history would hold {self.R + n - self.keep} samples per row, more than 2^31 - 1")
        out = self.stream.push(chunk)              # validates the chunk before any launch
        if n:
            need = self.S * self.C * (self.R + n - self.keep)
            if self.buf[1].numel() < need:
                self.buf[1] = torch.empty(max(need, 2 * self.buf[1].numel()), device=self.device)
            self.history = stream_history_(self.buf[1], self.history, self.h0, chunk, self.keep)
            self.buf.reverse()
            self.h0, self.R = self.keep, self.R + n
        return self._finish(out)

    @torch.no_grad()
    def close(self) -> CharacterizedOutput:
        return self._finish(self.stream.close())

    def _finish(self, out: StreamOutput) -> CharacterizedOutput:
        pk = self.stream.picker
        self.keep = max(self.keep, min(pk.first_pend[1], pk.F - 1) - self.ch.anchor)
        index, _, offsets = out.ppk
        rel = index - self.h0 if index.numel() else index
        return CharacterizedOutput(out, self.ch._run(self.history, rel, offsets))
