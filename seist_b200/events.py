"""Characterise picked events on continuous records (DESIGN §4.17): every P pick of a pick list through the polarity,
magnitude, back-azimuth and distance models.

The reference defines how these models see an event: `DataPreprocessor._cut_window` with 0 <= p_position_ratio <= 1
(training/preprocess.py:172-203) cuts `in_samples` with the first P pick at sample int(in_samples * p_position_ratio),
zero-filling what falls outside the trace, and `_normalize` (:224-242) normalises the window per channel.  Here the P
picks of a whole record, as the CSR `ContinuousAnnotator.pick_phases(...)["ppk"]` returns them, are cut straight into the
static inputs of the models' captured eval plans (`InferenceGraph`) by one kernel launch per batch of events
(`seist_event_windows`, csrc/stream.cu), and the outputs come back aligned index for index with the pick list.  The numpy
restatement of the cut is `oracle/event_ref.py`.  `EventCharacterizer.open_stream` does the same for the P picks of a
record streamed chunk by chunk, in the call that emits them (DESIGN §4.18), and `open_ragged_stream` / `open_gap_stream`
for streams whose stations advance at different rates (§4.20) or whose data have gaps (§4.23).  There is no CPU path.
"""
from __future__ import annotations

import ctypes
from typing import NamedTuple

import numpy as np
import torch

from . import _lib
from .infer import InferenceGraph
from .stream import (_I32_MAX, _MODES, ContinuousAnnotator, RaggedStreamOutput, Segments, StreamOutput, _dense, _flat, _prefix, _s,
                     _upload, check_segments)

_HISTORY_ROWS = 65535       # S * C rows of one seist_ragged_history launch (grid.y)

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


def segment_event_windows_(xs, record: torch.Tensor, segs: Segments, index: torch.Tensor, offsets: torch.Tensor, e0: int, window: int,
                           anchor: int, norm_mode: str = "std"):
    """event_windows_ zero-filling outside the pick's own annotated segment of `segs` (gap_segments of record) instead of
    outside [0, T); picks outside every annotated segment give zero rows."""
    _dense(record, (None, None, None), "record")
    S, C, T = record.shape
    if not 1 <= len(xs) <= MAX_MODELS:
        raise ValueError(f"1 to {MAX_MODELS} destinations, got {len(xs)}")
    for x in xs:
        _dense(x, (xs[0].shape[0], C, window), "event window batch", record.device)
    _check_picks(index, offsets, S, record.device)
    check_segments(segs, S, T, record.device)
    if not (1 <= window <= MAX_WINDOW and 0 <= anchor <= window and T < 2 ** 31 and e0 >= 0):
        raise ValueError(f"need 1 <= window <= {MAX_WINDOW}, 0 <= anchor <= window, T < 2^31 and e0 >= 0, got window {window}, "
                         f"anchor {anchor}, T {T}, e0 {e0}")
    G = len(segs.on)
    ptrs = (ctypes.c_void_p * MAX_MODELS)(*[x.data_ptr() for x in xs])
    _lib.check(_lib.lib().seist_segment_event_windows(record.data_ptr(), S, C, T, segs.pairs.data_ptr() if G else None,
                                                      segs.offsets.data_ptr(), segs.annotated.data_ptr() if G else None, G,
                                                      index.data_ptr(), index.numel(), offsets.data_ptr(), e0, xs[0].shape[0], window,
                                                      anchor, _MODES[norm_mode], ptrs, len(xs), _s()), "seist_segment_event_windows")
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
    def __call__(self, record: torch.Tensor, ppk, segments: Segments | None = None) -> dict:
        """With segments (`ContinuousAnnotator.segments(record)`), each pick's window is zero outside the pick's own
        annotated segment, and a pick outside every annotated segment gets a zero window (DESIGN §4.21)."""
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
        if segments is not None:
            check_segments(segments, S, T, self.device)
            record = record.contiguous()
            return self._batches(index.numel(), lambda xs, e0: segment_event_windows_(
                xs, record, segments, index, offsets, e0, self.window, self.anchor, self.norm_mode))
        return self._run(record.contiguous(), index, offsets)

    def _run(self, record: torch.Tensor, index: torch.Tensor, offsets: torch.Tensor) -> dict:
        return self._batches(index.numel(), lambda xs, e0: event_windows_(xs, record, index, offsets, e0, self.window, self.anchor,
                                                                          self.norm_mode))

    def _batches(self, M: int, cut) -> dict:
        """M events in batches: cut(xs, e0) writes every model's input for events e0 .., then each model replays."""
        out = {name: torch.empty((M,) if self.heads[name] == "reg" else (M, g.y.shape[1]), dtype=torch.float32, device=self.device)
               for name, g in self.graphs.items()}
        xs = [g.x for g in self.graphs.values()]
        for e0 in range(0, M, self.batch):
            cut(xs, e0)
            n = min(self.batch, M - e0)
            for name, g in self.graphs.items():
                y = g.replay()
                out[name][e0:e0 + n] = y[:n, 0] if self.heads[name] == "reg" else y[:n]
        return out

    def open_stream(self, annotator: ContinuousAnnotator, n_stations: int) -> "CharacterizedStream":
        """A record picked chunk by chunk by `annotator` (a dpk ContinuousAnnotator, thresholds and min_peak_dist set),
        every P pick characterised in the call that emits it (DESIGN §4.18)."""
        return CharacterizedStream(self, annotator, n_stations)

    def open_ragged_stream(self, annotator: ContinuousAnnotator, n_stations: int) -> "RaggedCharacterizedStream":
        """Stations that advance at different rates (`annotator.open_ragged_stream`), every P pick characterised in the call
        that emits it (DESIGN §4.20)."""
        return RaggedCharacterizedStream(self, annotator, n_stations)

    def open_gap_stream(self, annotator: ContinuousAnnotator, n_stations: int) -> "GapCharacterizedStream":
        """Stations whose data have gaps (`annotator.open_gap_stream`), every P pick characterised in the call that emits
        it, its window zero outside the pick's own segment (DESIGN §4.23)."""
        return GapCharacterizedStream(self, annotator, n_stations)


def _check_pair(ch: EventCharacterizer, ann: ContinuousAnnotator):
    """A characteriser and an annotator that can stream together (raises ValueError otherwise)."""
    dev = next(ann.model.parameters()).device
    if dev != ch.device:
        raise ValueError(f"the annotator's model is on {dev}, the characteriser's models on {ch.device}")
    if ann.in_channels != ch.in_channels:
        raise ValueError(f"the annotator takes {ann.in_channels} channels, the characteriser's models {ch.in_channels}")
    if ch.window - ch.anchor > ann.window:
        raise ValueError(f"the characteriser's window reaches {ch.window - ch.anchor} samples past the pick, more than the "
                         f"annotator's window ({ann.window}): a pick's event window would not be pushed yet when it closes")


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
        _check_pair(ch, ann)
        self.ch = ch
        self.stream = ann.open_stream(n_stations)
        self.S, self.C, self.device = self.stream.S, self.stream.C, self.stream.device
        self.buf = [torch.zeros(1, device=self.device), torch.zeros(1, device=self.device)]
        self.desc = torch.zeros(2 * self.S + 1, dtype=torch.int64, device=self.device)   # h0 (S,), off (S + 1,) of buf[0]
        self.history = self.buf[0][:0].view(self.S, self.C, 0)
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
        S, C = self.S, self.C
        hp = ragged_history_plan(np.full(S, self.h0), np.full(S, self.R), np.full(S, n), np.full(S, self.keep)) if n else None
        out = self.stream.push(chunk)              # validates the chunk before any launch
        if n:
            self.desc = push_history_(self.buf, self.desc, hp, chunk, n * np.arange(S + 1), C)   # the (S, C, n) chunk is packed
            self.h0, self.R = self.keep, self.R + n
            self.history = self.buf[0][:S * C * (self.R - self.h0)].view(S, C, self.R - self.h0)
        return self._finish(out)

    @torch.no_grad()
    def close(self) -> CharacterizedOutput:
        return self._finish(self.stream.close())

    def _finish(self, out: StreamOutput) -> CharacterizedOutput:
        pk = self.stream.picker
        self.keep = max(self.keep, int(min(pk.first_pend[1].min(), pk.F.min() - 1)) - self.ch.anchor)
        index, _, offsets = out.ppk
        rel = index - self.h0 if index.numel() else index
        return CharacterizedOutput(out, self.ch._run(self.history, rel, offsets))


# ---- ragged characterised streams: stations that advance at different rates (DESIGN §4.20) ----------------------------
def ragged_history_plan(h0, R, n, keep) -> dict:
    """The per-station history bookkeeping of one call of a RaggedCharacterizedStream, from the held samples [h0, R) of
    each station (S,), this call's push lengths n (S,) and the retention bounds keep (S,) of the previous call: a station
    with n > 0 holds [keep, R + n) after the call, one with n = 0 keeps [h0, R).  Returns numpy int64 arrays h0, R, len
    (S,) of the new histories and off (S + 1,), their exclusive prefix (station s packed as a (C, len) block at C * off[s])."""
    h0, R, n, keep = (np.asarray(v, dtype=np.int64).reshape(-1) for v in (h0, R, n, keep))
    if not (h0.shape == R.shape == n.shape == keep.shape) or (n < 0).any() or (h0 > R).any():
        raise ValueError(f"expected (S,) counts with h0 <= R and n >= 0, got h0 {h0.tolist()}, R {R.tolist()}, n {n.tolist()}")
    r1 = R + n
    h0_out = np.where(n > 0, keep, h0)
    if ((n > 0) & ((keep < h0) | (keep > r1))).any():
        raise ValueError(f"a retention bound outside the held samples: h0 {h0.tolist()}, keep {keep.tolist()}, R + n {r1.tolist()}")
    length = r1 - h0_out
    return {"h0": h0_out, "R": r1, "len": length, "off": _prefix(length)}


def _per_station(t: torch.Tensor, n: int, what: str, device):
    if not (t.is_cuda and t.dtype == torch.int64 and t.dim() == 1 and t.is_contiguous() and t.numel() == n and t.device == device):
        raise ValueError(f"{what}: expected a contiguous int64 CUDA tensor of shape ({n},) on {device}, "
                         f"got {tuple(t.shape)} {t.dtype} on {t.device}")


def ragged_history_(out: torch.Tensor, held: torch.Tensor, held_h0: torch.Tensor, held_off: torch.Tensor, chunk: torch.Tensor,
                    chunk_off: torch.Tensor, h0_out: torch.Tensor, out_off: torch.Tensor, C: int, max_len: int) -> torch.Tensor:
    """Write the packed histories (station s: samples [h0_out[s], ..) as a (C, len_s) block at C * out_off[s]) into the flat
    float32 buffer out, from the packed held histories (held_h0, held_off) followed by each station's block of the packed
    chunk (C * chunk_off[s]).  Per-station arrays are int64 on the device; max_len >= every len_s sizes the grid."""
    S = h0_out.numel()
    dev = held.device
    _flat(held, 0, "held histories", dev)
    _flat(chunk, 0, "packed chunk", dev)
    _flat(out, 0, "history buffer", dev)
    for t, what, k in ((held_h0, "held h0", S), (held_off, "held offsets", S + 1), (chunk_off, "chunk offsets", S + 1),
                       (h0_out, "h0_out", S), (out_off, "out offsets", S + 1)):
        _per_station(t, k, what, dev)
    if not (S >= 1 and S * int(C) <= 65535 and 0 <= int(max_len) <= _I32_MAX):
        raise ValueError(f"need 1 <= S, S * C <= 65535 and 0 <= max_len < 2^31, got S {S}, C {C}, max_len {max_len}")
    if out.data_ptr() in (held.data_ptr(), chunk.data_ptr()):
        raise ValueError("the history buffer must be distinct from the held histories and the chunk")
    _lib.check(_lib.lib().seist_ragged_history(held.data_ptr(), held_off.data_ptr(), held_h0.data_ptr(), held.numel(), chunk.data_ptr(),
                                               chunk_off.data_ptr(), chunk.numel(), h0_out.data_ptr(), out_off.data_ptr(), S, int(C),
                                               int(max_len), out.data_ptr(), out.numel(), _s()), "seist_ragged_history")
    return out


def push_history_(buf: list, desc: torch.Tensor, hp: dict, chunk: torch.Tensor, chunk_off, C: int) -> torch.Tensor:
    """One history step of a characterised stream: the histories planned by `ragged_history_plan` (hp) written into
    buf[1], grown when too small, from the held histories in buf[0] (device h0 (S,) and offsets (S + 1,) in desc) followed
    by each station's block of the packed chunk (C * chunk_off[s], host int64 (S + 1,)); then the two buffers swap.
    Returns the device h0 and offsets (2S + 1,) of the histories now in buf[0]."""
    S, dev = hp["h0"].size, desc.device
    need = C * int(hp["off"][-1])
    if buf[1].numel() < need:
        buf[1] = torch.empty(max(need, 2 * buf[1].numel()), device=dev)
    d = _upload(np.concatenate([hp["h0"], hp["off"], chunk_off]), dev)   # the history descriptors
    ragged_history_(buf[1], buf[0], desc[:S], desc[S:], chunk, d[2 * S + 1:], d[:S], d[S:2 * S + 1], C, int(hp["len"].max()))
    buf.reverse()
    return d[:2 * S + 1]


def ragged_event_windows_(xs, hist: torch.Tensor, hist_h0: torch.Tensor, hist_off: torch.Tensor, index: torch.Tensor,
                          offsets: torch.Tensor, e0: int, window: int, anchor: int, norm_mode: str = "std"):
    """event_windows_ cutting from packed histories (station s: a (C, len_s) block at C * hist_off[s] whose first sample is
    the global hist_h0[s]): every x in xs (B, C, window) gets events e0 .. e0 + B - 1 of the pick CSR, whose global
    indices are rebased on the device; zeros outside the station's history."""
    S = hist_h0.numel()
    dev = hist.device
    _flat(hist, 0, "histories", dev)
    _per_station(hist_h0, S, "history h0", dev)
    _per_station(hist_off, S + 1, "history offsets", dev)
    if not 1 <= len(xs) <= MAX_MODELS:
        raise ValueError(f"1 to {MAX_MODELS} destinations, got {len(xs)}")
    C = xs[0].shape[1] if xs[0].dim() == 3 else -1
    for x in xs:
        _dense(x, (xs[0].shape[0], C, window), "event window batch", dev)
    _check_picks(index, offsets, S, dev)
    if not (1 <= window <= MAX_WINDOW and 0 <= anchor <= window and e0 >= 0 and S >= 1):
        raise ValueError(f"need 1 <= window <= {MAX_WINDOW}, 0 <= anchor <= window and e0 >= 0, got window {window}, "
                         f"anchor {anchor}, e0 {e0}")
    ptrs = (ctypes.c_void_p * MAX_MODELS)(*[x.data_ptr() for x in xs])
    _lib.check(_lib.lib().seist_ragged_event_windows(hist.data_ptr(), hist_off.data_ptr(), hist_h0.data_ptr(), hist.numel(), S, C,
                                                     index.data_ptr(), index.numel(), offsets.data_ptr(), e0, xs[0].shape[0], window,
                                                     anchor, _MODES[norm_mode], ptrs, len(xs), _s()), "seist_ragged_event_windows")
    return xs


class RaggedCharacterizedOutput(NamedTuple):
    """One call of a RaggedCharacterizedStream: the RaggedStream's RaggedStreamOutput and {name: outputs} for its P picks,
    row i for pick i of `out.ppk`."""
    out: RaggedStreamOutput
    events: dict


class RaggedCharacterizedStream:
    """`EventCharacterizer.open_ragged_stream(annotator, n_stations)`: `push(chunks)` with S float32 (C, n_s) tensors, any
    n_s >= 0, then `close()`, each -> RaggedCharacterizedOutput.  Station s's events, concatenated over the calls, equal
    `ch(rec_s[None], annotator.pick_phases(annotator.annotate(rec_s[None]))["ppk"])` of its own record bit for bit, each in
    the call that emits its pick (DESIGN §4.20).  Each station keeps the §4.18 history on its own counts: the raw samples
    [h0_s, R_s), h0_s the retention bound max(0, min(first pending P candidate, F_s - 1) - anchor) of the call before the
    station's last non-empty push.  The histories are packed back to back in one of two flat device buffers, their h0 and
    offsets in a small device array.  `held_samples` = R - h0 per station ((S,) int64)."""

    def __init__(self, ch: EventCharacterizer, ann: ContinuousAnnotator, n_stations: int):
        _check_pair(ch, ann)
        self.ch = ch
        self.stream = ann.open_ragged_stream(n_stations)
        self.S, self.C, self.device = self.stream.S, self.stream.C, self.stream.device
        self.buf = [torch.zeros(1, device=self.device), torch.zeros(1, device=self.device)]
        self.desc = torch.zeros(2 * self.S + 1, dtype=torch.int64, device=self.device)   # h0 (S,), off (S + 1,) of buf[0]
        self.h0 = np.zeros(self.S, np.int64)
        self.R = np.zeros(self.S, np.int64)
        self.keep = np.zeros(self.S, np.int64)       # the retention bounds after the last call

    @property
    def closed(self) -> bool:
        return self.stream.closed

    @property
    def forwards(self) -> int:
        return self.stream.forwards

    @property
    def held_samples(self) -> np.ndarray:
        return self.R - self.h0

    @torch.no_grad()
    def push(self, chunks) -> RaggedCharacterizedOutput:
        plan, chunk = self.stream._prepare(chunks)                # validates the chunks before any launch
        n = plan["r1"] - plan["r0"]
        hp = ragged_history_plan(self.h0, self.R, n, self.keep)
        if (hp["len"] > _I32_MAX).any():
            s = np.nonzero(hp["len"] > _I32_MAX)[0].tolist()
            raise ValueError(f"the histories of stations {s} would hold {hp['len'][s].tolist()} samples, more than 2^31 - 1")
        out = self.stream._call(plan, chunk, False)
        if n.any():
            self.desc = push_history_(self.buf, self.desc, hp, chunk, plan["chunk_off"], self.C)
            self.h0 = hp["h0"]
        self.R = hp["R"]
        return self._finish(out)

    @torch.no_grad()
    def close(self) -> RaggedCharacterizedOutput:
        return self._finish(self.stream.close())

    def _finish(self, out: RaggedStreamOutput) -> RaggedCharacterizedOutput:
        pk, ch, S = self.stream.picker, self.ch, self.S
        self.keep = np.maximum(self.keep, np.minimum(pk.first_pend[1], pk.F - 1) - ch.anchor)
        index, _, offsets = out.ppk
        hist, h0, off = self.buf[0], self.desc[:S], self.desc[S:]
        return RaggedCharacterizedOutput(out, ch._batches(index.numel(), lambda xs, e0: ragged_event_windows_(
            xs, hist, h0, off, index, offsets, e0, ch.window, ch.anchor, ch.norm_mode)))


# ---- characterised streams with data gaps (DESIGN §4.23) ----------------------------------------------------------------
def gap_history_keep(keep, seg_on, R, first_pend, F, anchor: int) -> np.ndarray:
    """The retention bounds (S,) after one call of a GapCharacterizedStream, from the bounds keep (S,) before it and the
    state after it: each station's open segment's first sample seg_on (-1 when the station ends the call in a gap), its
    samples pushed R, and first_pend / F, the first pending P candidate and the final count of its open segment's picker
    row (station indices).  §4.20's rule on the open segment, clamped at its first sample because no window reads below
    its own segment: max(keep, seg_on, min(first_pend, F - 1) - anchor); R for a station in a gap, which releases its
    history at its next non-empty push.  Feeds `ragged_history_plan`."""
    keep, seg_on, R, first_pend, F = (np.asarray(v, dtype=np.int64).reshape(-1) for v in (keep, seg_on, R, first_pend, F))
    if not (keep.shape == seg_on.shape == R.shape == first_pend.shape == F.shape):
        raise ValueError(f"expected (S,) arrays, got {[v.shape for v in (keep, seg_on, R, first_pend, F)]}")
    k = np.maximum(np.maximum(keep, seg_on), np.minimum(first_pend, F - 1) - int(anchor))
    return np.where(seg_on >= 0, k, R)


def gap_event_windows_(xs, hist: torch.Tensor, hist_h0: torch.Tensor, hist_off: torch.Tensor, pos_station: torch.Tensor,
                       pos_on: torch.Tensor, pos_end: torch.Tensor, pos_off: torch.Tensor, index: torch.Tensor, e0: int, window: int,
                       anchor: int, norm_mode: str = "std"):
    """ragged_event_windows_ for a gapped stream: event e is a pick of position q (the last with pos_off[q] <= e), whose
    station and global segment [on, end] are pos_station / pos_on / pos_end[q] ((n_pos,) int64 on the device); zeros
    outside [on, end] ∩ the station's history, so each window equals segment_event_windows_'s on the whole record."""
    S = hist_h0.numel()
    dev = hist.device
    _flat(hist, 0, "histories", dev)
    _per_station(hist_h0, S, "history h0", dev)
    _per_station(hist_off, S + 1, "history offsets", dev)
    n_pos = pos_station.numel()
    for t, what in ((pos_station, "position stations"), (pos_on, "position segment starts"), (pos_end, "position segment ends")):
        _per_station(t, n_pos, what, dev)
    if not 1 <= len(xs) <= MAX_MODELS:
        raise ValueError(f"1 to {MAX_MODELS} destinations, got {len(xs)}")
    C = xs[0].shape[1] if xs[0].dim() == 3 else -1
    for x in xs:
        _dense(x, (xs[0].shape[0], C, window), "event window batch", dev)
    _check_picks(index, pos_off, n_pos, dev)
    if not (1 <= window <= MAX_WINDOW and 0 <= anchor <= window and e0 >= 0 and S >= 1 and 1 <= n_pos <= _I32_MAX):
        raise ValueError(f"need 1 <= window <= {MAX_WINDOW}, 0 <= anchor <= window, e0 >= 0 and 1 <= n_pos < 2^31, got window "
                         f"{window}, anchor {anchor}, e0 {e0}, n_pos {n_pos}")
    ptrs = (ctypes.c_void_p * MAX_MODELS)(*[x.data_ptr() for x in xs])
    _lib.check(_lib.lib().seist_gap_event_windows(hist.data_ptr(), hist_off.data_ptr(), hist_h0.data_ptr(), hist.numel(), S, C,
                                                  pos_station.data_ptr(), pos_on.data_ptr(), pos_end.data_ptr(), pos_off.data_ptr(), n_pos,
                                                  index.data_ptr(), index.numel(), e0, xs[0].shape[0], window, anchor, _MODES[norm_mode],
                                                  ptrs, len(xs), _s()), "seist_gap_event_windows")
    return xs


class GapCharacterizedStream:
    """`EventCharacterizer.open_gap_stream(annotator, n_stations)`: `push(chunks)` and `close()` take what `GapStream`'s
    take (S float32 (C, n_s) tensors, any n_s >= 0, NaN / Inf marking gap samples), each -> RaggedCharacterizedOutput
    whose `out` is the GapStream's output.  Station s's events, concatenated over the calls, equal `ch(rec_s[None], ppk,
    segments=segs)` with `segs = annotator.segments(rec_s[None])` and `ppk = annotator.pick_phases(annotator.annotate(
    rec_s[None], segments=segs), segments=segs)["ppk"]` bit for bit, each in the call that emits its pick (DESIGN §4.23).
    Each station keeps the raw samples [h0_s, R_s), h0_s the `gap_history_keep` bound of the call before its last
    non-empty push; the histories are packed as in RaggedCharacterizedStream.  `held_samples` = R - h0 per station ((S,)
    int64)."""

    def __init__(self, ch: EventCharacterizer, ann: ContinuousAnnotator, n_stations: int):
        _check_pair(ch, ann)
        if int(n_stations) * ch.in_channels > _HISTORY_ROWS:
            raise ValueError(f"{n_stations} stations of {ch.in_channels} channels: the history kernel takes at most "
                             f"{_HISTORY_ROWS} station channels (S * C)")
        self.ch = ch
        self.stream = ann.open_gap_stream(n_stations)
        self.S, self.C, self.device = self.stream.S, self.stream.C, self.stream.device
        self.buf = [torch.zeros(1, device=self.device), torch.zeros(1, device=self.device)]
        self.desc = torch.zeros(2 * self.S + 1, dtype=torch.int64, device=self.device)   # h0 (S,), off (S + 1,) of buf[0]
        self.h0 = np.zeros(self.S, np.int64)
        self.R = np.zeros(self.S, np.int64)
        self.keep = np.zeros(self.S, np.int64)       # the retention bounds after the last call

    @property
    def closed(self) -> bool:
        return self.stream.closed

    @property
    def forwards(self) -> int:
        return self.stream.forwards

    @property
    def held_samples(self) -> np.ndarray:
        return self.R - self.h0

    @torch.no_grad()
    def push(self, chunks) -> RaggedCharacterizedOutput:
        n = self.stream._lengths(chunks)                          # validates the chunks before any launch
        hp = ragged_history_plan(self.h0, self.R, n, self.keep)
        if (hp["len"] > _I32_MAX).any():
            s = np.nonzero(hp["len"] > _I32_MAX)[0].tolist()
            raise ValueError(f"the histories of stations {s} would hold {hp['len'][s].tolist()} samples, more than 2^31 - 1")
        plan, chunk, chunk_off = self.stream._prepare(chunks)
        out, where = self.stream._call(plan, chunk, chunk_off)
        S = self.S
        hist = [hp["h0"], hp["off"], chunk_off] if n.any() else []
        dev = _upload(np.concatenate(hist + [where["station"], where["on"], where["end"]]), self.device)   # the call's descriptors
        if n.any():
            need = self.C * int(hp["off"][-1])
            if self.buf[1].numel() < need:
                self.buf[1] = torch.empty(max(need, 2 * self.buf[1].numel()), device=self.device)
            ragged_history_(self.buf[1], self.buf[0], self.desc[:S], self.desc[S:], chunk, dev[2 * S + 1:3 * S + 2], dev[:S],
                            dev[S:2 * S + 1], self.C, int(hp["len"].max()))
            self.buf.reverse()
            self.desc = dev[:2 * S + 1]
            self.h0 = hp["h0"]
        self.R = hp["R"]
        return self._finish(out, where, dev[3 * S + 2 if n.any() else 0:])

    @torch.no_grad()
    def close(self) -> RaggedCharacterizedOutput:
        out, where = self.stream._close()
        dev = _upload(np.concatenate([where["station"], where["on"], where["end"]]), self.device)
        return self._finish(out, where, dev)

    def _finish(self, out: RaggedStreamOutput, where: dict, table: torch.Tensor) -> RaggedCharacterizedOutput:
        gs, ch, S = self.stream, self.ch, self.S
        pk, state = gs.picker, gs.state
        row = 2 * np.arange(S) + gs.flip                       # each station's open-segment row after the call
        self.keep = gap_history_keep(self.keep, state["seg_on"], state["R"], pk.first_pend[1][row], pk.F[row], ch.anchor)
        index = out.ppk[0]
        n_pos = where["station"].size
        st, on, end = table[:n_pos], table[n_pos:2 * n_pos], table[2 * n_pos:3 * n_pos]
        hist, h0, off, pos_off = self.buf[0], self.desc[:S], self.desc[S:], where["pos_off"]
        return RaggedCharacterizedOutput(out, ch._batches(index.numel(), lambda xs, e0: gap_event_windows_(
            xs, hist, h0, off, st, on, end, pos_off, index, e0, ch.window, ch.anchor, ch.norm_mode)))
