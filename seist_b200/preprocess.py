"""Input side on the device (SURVEY §8f-3): the training-time augmentation and window cut, per-trace normalisation, the
dpk soft labels and the metric targets.

The reference does both per waveform in numpy inside the DataLoader workers (`training/preprocess.py`:
`DataPreprocessor._normalize` :224-242, `_generate_soft_label` :544-683).  At the throughput of the fused training step
eight worker processes cannot feed one GPU; here a raw (N, C, L) batch and the (N, K) phase indices are turned into the
model input and the (N, 3, L) label tensor by two kernel launches on the device the step runs on.  `DevicePreprocessor`
does the whole of `DataPreprocessor.process` (:501-542), augmentation included, before the labels.  No CPU path.
"""
from __future__ import annotations

import ctypes

import torch
import torch.distributed as dist

from . import _lib

ABSENT = -10_000_000                       # "no phase" padding of the (N, K) index tensors
_MODES = {"": 0, "std": 1, "max": 2}
_SHAPES = {"gaussian": 0, "triangle": 1, "box": 2, "sigmoid": 3}
MAX_PHASES = 8                             # phase list entries (dpk_soft_labels takes K <= 8)
MAX_SAMPLES = 16384                        # raw trace length of process_batch: a 3-channel trace fills 192 KB of shared memory


def _s() -> int:
    return torch.cuda.current_stream().cuda_stream


def normalize_(x: torch.Tensor, mode: str = "std") -> torch.Tensor:
    """In-place `_normalize(data, mode)` of every (n, c) trace of a contiguous CUDA fp32 (N, C, L) batch."""
    if mode not in _MODES:
        raise ValueError(f"Supported mode: 'max','std', got '{mode}'")       # the reference's message
    if not x.is_cuda or x.dtype != torch.float32 or not x.is_contiguous() or x.dim() != 3:
        raise RuntimeError("seist_b200.preprocess.normalize_ needs a contiguous CUDA float32 (N, C, L) tensor (no CPU path)")
    n, c, l = x.shape
    _lib.check(_lib.lib().seist_normalize(x.data_ptr(), n * c, l, _MODES[mode], _s()), "seist_normalize")
    return x


def dpk_soft_labels(ppks: torch.Tensor, spks: torch.Tensor, length: int, soft_label_width: int,
                    soft_label_shape: str = "gaussian", coda_ratio: float = 1.4) -> torch.Tensor:
    """(N, K) int64 P / S sample indices (pad missing phases with `ABSENT`) -> (N, 3, length) float32 labels
    [det, ppk, spk] as `DataPreprocessor._generate_soft_label` builds them.  The sigmoid shape needs a width of at least 2
    (the reference divides by width // 2)."""
    if soft_label_shape not in _SHAPES:
        raise NotImplementedError(f"Unsupported label shape: '{soft_label_shape}'")
    if soft_label_shape == "sigmoid" and int(soft_label_width) < 2:
        raise ValueError(f"sigmoid soft labels need soft_label_width >= 2, got {soft_label_width}")
    if not ppks.is_cuda or ppks.shape != spks.shape or ppks.dim() != 2:
        raise RuntimeError("dpk_soft_labels needs two CUDA (N, K) index tensors of the same shape (no CPU path)")
    p = ppks.to(torch.int64).contiguous()
    s = spks.to(device=p.device, dtype=torch.int64).contiguous()
    n, k = p.shape
    out = torch.empty(n, 3, length, dtype=torch.float32, device=p.device)
    _lib.check(_lib.lib().seist_dpk_labels(p.data_ptr(), s.data_ptr(), n, k, length, int(soft_label_width), _SHAPES[soft_label_shape],
                                           float(coda_ratio), out.data_ptr(), _s()), "seist_dpk_labels")
    return out


def metric_targets(ppks: torch.Tensor, spks: torch.Tensor, max_event_num: int, soft_label_width: int, in_samples: int,
                   coda_ratio: float, expected_num: int) -> dict:
    """`get_targets_for_metrics` (:761-804) for the tasks det / ppk / spk from the output phase lists of
    `DevicePreprocessor.process_batch` (sorted, padded with ABSENT), in torch on their device (no kernel, no host sync):

      * "ppk" / "spk": (N, max(max_event_num, K)) int64, the list padded with int(-1e7) (= ABSENT);
      * "det": (N, 2 E) int64 [start, end, ...], E = max(expected_num, 2 K): the (P, S) pairs after `_pad_phases` with
        padding `soft_label_width`, start clipped to [0, in_samples], end = int(S + coda_ratio (S - P)), padded with [1, 0].
    These are the tensors `postprocess.StepCounters.update` takes.  Where the reference raises (a list longer than
    max_event_num) the list is kept whole; where it returns more than expected_num pairs the extra pairs are kept and every
    trace is padded to E pairs."""
    n, k = ppks.shape
    dev = ppks.device
    width = max(int(max_event_num), k)
    pick = {}
    for name, t in (("ppk", ppks), ("spk", spks)):
        out = torch.full((n, width), ABSENT, dtype=torch.int64, device=dev)
        out[:, :k] = t
        pick[name] = out
    valid_p, valid_s = ppks > ABSENT, spks > ABSENT
    n_p, n_s = valid_p.sum(1), valid_s.sum(1)
    big = torch.iinfo(torch.int64).max
    p_sorted = torch.where(valid_p, ppks, big).sort(1).values
    s_sorted = torch.where(valid_s, spks, big).sort(1).values
    # _pad_phases: idx = the largest i such that the first i sorted P all precede the last i sorted S, pairwise
    idx = torch.zeros(n, dtype=torch.int64, device=dev)
    alive = torch.ones(n, dtype=torch.bool, device=dev)
    ar = torch.arange(k, device=dev)
    for i in range(k):
        s_pos = (n_s - i - 1).unsqueeze(1) + ar.unsqueeze(0)             # S index paired with P index a <= i
        s_val = s_sorted.gather(1, s_pos.clamp(0, k - 1))
        ok = ((p_sorted < s_val) | (ar > i).unsqueeze(0)).all(1) & (i < torch.minimum(n_p, n_s)) & alive
        idx = idx + ok.long()
        alive = ok
    pad = abs(int(soft_label_width))
    lead = n_s - idx                                                      # leading P padding entries
    m = lead + n_p                                                        # pairs
    e = max(int(expected_num), 2 * k)
    j = torch.arange(e, device=dev).unsqueeze(0)
    p_idx = (j - lead.unsqueeze(1)).clamp(0, k - 1)
    pp = torch.where(j < lead.unsqueeze(1), -pad, p_sorted.gather(1, p_idx))
    ss = torch.where(j < n_s.unsqueeze(1), s_sorted.gather(1, j.clamp(max=k - 1)), in_samples + pad)
    st = pp.clamp(0, in_samples)
    et = (ss.double() + float(coda_ratio) * (ss - pp).double()).long()   # int(): truncation toward zero
    live = j < m.unsqueeze(1)
    det = torch.stack([torch.where(live, st, 1), torch.where(live, et, 0)], dim=2).reshape(n, 2 * e)
    return {"det": det, "ppk": pick["ppk"], "spk": pick["spk"]}


class DevicePreprocessor:
    """`DataPreprocessor.process(event, augmentation)` (training/preprocess.py:501-542) for a whole batch on the device:
    `_is_noise`, `_pad_phases` with `min_event_gap`, `_data_augmentation` (:432-499) for the traces whose flag is set,
    `_cut_window` (:172-222) and `_normalize`, in two kernel launches (csrc/augment.cu) with no host synchronisation, so
    the call can be captured into a CUDA graph.  Feed the output phase lists to `dpk_soft_labels` for the loss targets
    and to `metric_targets` for the metric targets.

    The constructor takes the keyword names of the reference's `DataPreprocessor.__init__`; `p_position_ratio` in [0, 1]
    zeroes `add_event_rate`, `shift_event_rate` and `generate_noise_rate` as :113-130 does.  Randomness comes from a
    counter-based generator on the device (`tests/augment_ref.py::CounterDraws` restates it): the draws of every
    augmentation branch follow the reference's order and ranges, not numpy's streams.  The seed is a device scalar
    advanced by every call, so graph replays draw new augmentations; it starts from `torch.initial_seed()` and the
    distributed rank, and `state_dict()` / `load_state_dict()` checkpoint it.

    Where the reference raises, the device gives a defined result instead: an event with more P than S picks is noise;
    with `p_position_ratio` in [0, 1] an event without P is cut from sample 0.
    """

    def __init__(self, data_channels, sampling_rate: int, in_samples: int, min_snr: float = -float("inf"),
                 p_position_ratio: float = -1, coda_ratio: float = 2.0, norm_mode: str = "std", add_event_rate: float = 0.0,
                 add_noise_rate: float = 0.4, add_gap_rate: float = 0.4, drop_channel_rate: float = 0.4,
                 scale_amplitude_rate: float = 0.4, pre_emphasis_rate: float = 0.4, pre_emphasis_ratio: float = 0.97,
                 max_event_num: int = 1, generate_noise_rate: float = 0.05, shift_event_rate: float = 0.2,
                 mask_percent: int = 0, noise_percent: int = 0, min_event_gap_sec: float = 0.5,
                 soft_label_shape: str = "gaussian", soft_label_width: int = 25, dtype=None):
        if norm_mode not in _MODES:
            raise ValueError(f"Supported mode: 'max','std', got '{norm_mode}'")
        if soft_label_shape not in _SHAPES:
            raise NotImplementedError(f"Unsupported label shape: '{soft_label_shape}'")
        self.data_channels = data_channels
        self.sampling_rate, self.in_samples = int(sampling_rate), int(in_samples)
        self.min_snr, self.p_position_ratio, self.coda_ratio, self.norm_mode = min_snr, p_position_ratio, coda_ratio, norm_mode
        self.add_event_rate, self.add_noise_rate, self.add_gap_rate = add_event_rate, add_noise_rate, add_gap_rate
        self.drop_channel_rate, self.scale_amplitude_rate = drop_channel_rate, scale_amplitude_rate
        self.pre_emphasis_rate, self.pre_emphasis_ratio = pre_emphasis_rate, pre_emphasis_ratio
        self.max_event_num, self.generate_noise_rate, self.shift_event_rate = int(max_event_num), generate_noise_rate, shift_event_rate
        self.mask_percent, self.noise_percent = int(mask_percent), int(noise_percent)
        self.min_event_gap = int(min_event_gap_sec * self.sampling_rate)
        if 0 <= self.p_position_ratio <= 1:
            self.add_event_rate = self.shift_event_rate = self.generate_noise_rate = 0.0
        self.soft_label_shape, self.soft_label_width = soft_label_shape, int(soft_label_width)
        if self.in_samples < 1 or self.max_event_num > MAX_PHASES:
            raise ValueError(f"DevicePreprocessor: in_samples >= 1 and max_event_num <= {MAX_PHASES}")
        if (self.mask_percent > 0 or self.noise_percent > 0) and self.sampling_rate // 2 < 1:
            raise ValueError("DevicePreprocessor: mask / noise windows need sampling_rate >= 2")
        self.seed = None

    @classmethod
    def from_args(cls, args, sampling_rate: int, channels) -> "DevicePreprocessor":
        """From the reference's `main.py` arguments, as `SeismicDataset.__init__` builds its preprocessor (:883-907)."""
        return cls(data_channels=channels, sampling_rate=sampling_rate, in_samples=args.in_samples, min_snr=args.min_snr,
                   coda_ratio=args.coda_ratio, norm_mode=args.norm_mode, p_position_ratio=args.p_position_ratio,
                   add_event_rate=args.add_event_rate, add_noise_rate=args.add_noise_rate, add_gap_rate=args.add_gap_rate,
                   drop_channel_rate=args.drop_channel_rate, scale_amplitude_rate=args.scale_amplitude_rate,
                   pre_emphasis_rate=args.pre_emphasis_rate, pre_emphasis_ratio=args.pre_emphasis_ratio,
                   max_event_num=args.max_event_num, generate_noise_rate=args.generate_noise_rate,
                   shift_event_rate=args.shift_event_rate, mask_percent=args.mask_percent, noise_percent=args.noise_percent,
                   min_event_gap_sec=args.min_event_gap, soft_label_shape=args.label_shape,
                   soft_label_width=int(args.label_width * sampling_rate))

    @staticmethod
    def _initial_seed() -> int:
        """Follows torch.manual_seed() and differs per rank (its own constant: not the dropout counter's start)."""
        rank = dist.get_rank() if (dist.is_available() and dist.is_initialized()) else 0
        z = (torch.initial_seed() * 0xA24BAED4963EE407 + (rank + 1) * 0x9FB21C651E98DF25) & ((1 << 64) - 1)
        z ^= z >> 31
        return z & ((1 << 62) - 1)

    def _seed_on(self, device) -> torch.Tensor:
        if self.seed is None or self.seed.device != device:
            old = None if self.seed is None else int(self.seed.item())
            self.seed = torch.full((1,), self._initial_seed() if old is None else old, dtype=torch.int64, device=device)
        return self.seed

    def state_dict(self) -> dict:
        return {"seed": None if self.seed is None else int(self.seed.item())}

    def load_state_dict(self, state: dict, device=None):
        if state.get("seed") is None:
            self.seed = None
            return
        value = int(state["seed"]) & ((1 << 62) - 1)
        dev = torch.device(device) if device is not None else (self.seed.device if self.seed is not None else torch.device("cuda"))
        if self.seed is not None and self.seed.device == dev:
            self.seed.fill_(value)          # in place: a captured CUDA graph keeps reading this scalar
        else:
            self.seed = torch.full((1,), value, dtype=torch.int64, device=dev)

    def expected_det_num(self) -> int:
        """`expected_num` of `get_targets_for_metrics` (:793)."""
        return (self.max_event_num + int(bool(self.add_event_rate)) + int(bool(self.shift_event_rate))
                + int(0 <= self.p_position_ratio <= 1))

    def out_phases(self, k: int) -> int:
        """Width of the output phase lists for inputs of width k: add-event can grow a list up to max_event_num."""
        return max(k, self.max_event_num) if self.add_event_rate > 0 else k

    def _cfg(self) -> _lib.SeistAugCfg:
        return _lib.SeistAugCfg(
            generate_noise_rate=self.generate_noise_rate, add_event_rate=self.add_event_rate,
            shift_event_rate=self.shift_event_rate, drop_channel_rate=self.drop_channel_rate,
            scale_amplitude_rate=self.scale_amplitude_rate, pre_emphasis_rate=self.pre_emphasis_rate,
            add_noise_rate=self.add_noise_rate, add_gap_rate=self.add_gap_rate, coda_ratio=self.coda_ratio,
            min_snr=self.min_snr, p_position_ratio=self.p_position_ratio, pre_emphasis_ratio=self.pre_emphasis_ratio,
            in_samples=self.in_samples, min_event_gap=self.min_event_gap, max_event_num=self.max_event_num,
            norm_mode=_MODES[self.norm_mode], mask_percent=self.mask_percent, noise_percent=self.noise_percent,
            window=max(self.sampling_rate // 2, 1))

    def process_batch(self, data: torch.Tensor, ppks: torch.Tensor, spks: torch.Tensor, snr: torch.Tensor = None,
                      augment: torch.Tensor = None):
        """data (N, C, Lin) float32 raw traces (3 <= Lin <= 16384), ppks / spks (N, K) int64 sample indices padded with
        ABSENT, snr (N, S) or None (no trace is noise by SNR), augment (N,) bool or None (every trace augmented), all on
        one CUDA device.  Returns (x (N, C, in_samples) float32, ppks_out, spks_out (N, out_phases(K)) int64 sorted and
        padded with ABSENT, cleared (N,) bool: `_is_noise` or the generated noise cleared the event)."""
        if not data.is_cuda or data.dtype != torch.float32 or data.dim() != 3:
            raise RuntimeError("process_batch needs a CUDA float32 (N, C, Lin) tensor (no CPU path)")
        n, c, lin = data.shape
        if not 3 <= lin <= MAX_SAMPLES:
            raise ValueError(f"process_batch: raw length {lin} outside [3, {MAX_SAMPLES}]")
        if ppks.dim() != 2 or ppks.shape != spks.shape or ppks.shape[0] != n or not ppks.is_cuda or not spks.is_cuda:
            raise RuntimeError("process_batch needs two CUDA (N, K) index tensors of the same shape")
        k = ppks.shape[1]
        k_out = self.out_phases(k)
        if not 1 <= k or k_out > MAX_PHASES:
            raise ValueError(f"process_batch: K = {k} phases (plus add-event up to max_event_num) must stay <= {MAX_PHASES}")
        if (self.mask_percent > 0 or self.noise_percent > 0) and lin // max(self.sampling_rate // 2, 1) > 1024:
            raise ValueError("process_batch: more than 1024 mask / noise windows per trace")
        if n == 0:
            raise ValueError("process_batch: empty batch")
        dev = data.device
        data = data.contiguous()
        p = ppks.to(device=dev, dtype=torch.int64).contiguous()
        s = spks.to(device=dev, dtype=torch.int64).contiguous()
        snr_t, n_snr = None, 0
        if snr is not None:
            snr_t = snr.to(device=dev, dtype=torch.float64).reshape(n, -1).contiguous()
            n_snr = snr_t.shape[1]
        aug_t = None
        if augment is not None:
            aug_t = augment.to(device=dev, dtype=torch.bool).reshape(n).contiguous()
        seed = self._seed_on(dev)
        lib = _lib.lib()
        x = torch.empty(n, c, self.in_samples, dtype=torch.float32, device=dev)
        p_out = torch.empty(n, k_out, dtype=torch.int64, device=dev)
        s_out = torch.empty(n, k_out, dtype=torch.int64, device=dev)
        cleared = torch.empty(n, dtype=torch.bool, device=dev)
        work = torch.empty(n * lib.seist_aug_recipe_bytes(), dtype=torch.uint8, device=dev)
        cfg = self._cfg()
        _lib.check(lib.seist_augment(data.data_ptr(), n, c, lin, p.data_ptr(), s.data_ptr(), k,
                                     None if snr_t is None else snr_t.data_ptr(), n_snr,
                                     None if aug_t is None else aug_t.data_ptr(), ctypes.byref(cfg), seed.data_ptr(),
                                     x.data_ptr(), p_out.data_ptr(), s_out.data_ptr(), k_out, cleared.data_ptr(),
                                     work.data_ptr(), work.numel(), _s()), "seist_augment")
        _lib.check(lib.seist_advance_seed(seed.data_ptr(), _s()), "seist_advance_seed")
        return x, p_out, s_out, cleared

    def labels(self, ppks_out: torch.Tensor, spks_out: torch.Tensor) -> torch.Tensor:
        """(N, 3, in_samples) [det, ppk, spk] loss targets of the dpk task from the output phase lists."""
        return dpk_soft_labels(ppks_out, spks_out, self.in_samples, self.soft_label_width, self.soft_label_shape,
                               self.coda_ratio)

    def metric_targets(self, ppks_out: torch.Tensor, spks_out: torch.Tensor) -> dict:
        """`get_targets_for_metrics` for det / ppk / spk, see the module-level `metric_targets`."""
        return metric_targets(ppks_out, spks_out, self.max_event_num, self.soft_label_width, self.in_samples,
                              self.coda_ratio, self.expected_det_num())
