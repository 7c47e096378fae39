"""CPU oracle (TEST INFRASTRUCTURE) of the training-time input pipeline: the reference's `DataPreprocessor.process`
(training/preprocess.py:501-542) with `_data_augmentation` (:432-499), every transform it calls and `_cut_window`
(:172-222), restated in numpy behind a draw source, plus the sigmoid soft-label window (:586-597) and the metric targets
of `get_targets_for_metrics` (:761-804).

Two draw sources make the same calls in the same order:
  * `NumpyDraws`   - exactly the reference's `np.random.*` calls; seeded with `np.random.seed` this reproduces the reference
                     bit for bit (tests/test_cpu_augment.py against tests/golden/reference_augmentation.pt);
  * `CounterDraws` - what seist_b200/csrc/augment.cu draws on the device: uniforms from `rng_u64` (oracle/plan_interp.py,
                     csrc/common.cuh) on a per-trace counter, selection sampling for the mask / noise windows and counter
                     normals (Box-Muller on a hash of (seed, trace, channel, sample)).
Where the reference raises (an event without P under `p_position_ratio`, more P than S picks) the restatement follows
the device's documented result instead (seist_b200/preprocess.py::DevicePreprocessor).
"""
import math

import numpy as np

from oracle import preprocess_ref as PR
from oracle.plan_interp import rng_u64

ABSENT = -10_000_000
STREAM_DRAW = 0x41554700                 # csrc/augment.cu AUG_STREAM_DRAW / AUG_STREAM_NORMAL (no plan uses these ids)
STREAM_NORMAL = 0x41554710
NOISE_FILL, NOISE_ADD, NOISE_WINDOW = 0, 1, 2     # normal streams of generate-noise, add-noise and the noise windows


# ---- draw sources --------------------------------------------------------------------------------------------------
class NumpyDraws:
    """The reference's own global-state numpy calls, in its order (seed with np.random.seed before `process`)."""

    def random(self):
        return np.random.random()

    def randint(self, a, b):
        return np.random.randint(a, b)

    def uniform(self, a, b):
        return np.random.uniform(a, b)

    def choice_range(self, a, b):           # np.random.choice(range(a, b))
        return np.random.choice(range(a, b))

    def choice(self, cands):
        return np.random.choice(cands)

    def windows(self, n, k):                # np.random.choice(range(n), k, replace=False)
        return np.random.choice(range(n), k, replace=False)

    def normal(self, kind, chans, start, stop):
        return np.random.randn(len(chans), stop - start)


def counter_normal(seed: int, stream: int, q: np.ndarray) -> np.ndarray:
    """Box-Muller in double on one 64-bit hash: u1 = (hi + 1) / 2^32 in (0, 1], u2 = lo / 2^32."""
    h = rng_u64(seed, stream, q)
    u1 = ((h >> np.uint64(32)) + np.uint64(1)).astype(np.float64) * 2.0 ** -32
    u2 = (h & np.uint64(0xFFFFFFFF)).astype(np.float64) * 2.0 ** -32
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(6.283185307179586 * u2)


def normal_index(trace: int, channels: int, c, i):
    """Counter of the normal at (trace, channel c, sample i): ((trace * C + c) << 16) + i."""
    return ((np.uint64(trace * channels) + np.asarray(c, np.uint64)) << np.uint64(16)) + np.asarray(i, np.uint64)


class CounterDraws:
    """The device's draws for trace `trace` of a batch at seed `seed`: the k-th uniform of the trace is the top 53 bits of
    rng_u64(seed, STREAM_DRAW, (trace << 32) + k); randint(a, b) = a + floor(u (b - a)) (a when b <= a), uniform(a, b) =
    a + u (b - a)."""

    def __init__(self, seed: int, trace: int, channels: int):
        self.seed, self.n, self.C, self.k = int(seed), int(trace), int(channels), 0
        self._buf, self._pos = [], 0

    def _u(self) -> float:
        if self._pos == len(self._buf):      # 64 hashes per numpy call
            q = (np.uint64(self.n) << np.uint64(32)) + np.arange(self.k, self.k + 64, dtype=np.uint64)
            self._buf, self._pos = [int(v) for v in rng_u64(self.seed, STREAM_DRAW, q)], 0
        h = self._buf[self._pos]
        self._pos += 1
        self.k += 1
        return float(h >> 11) * 2.0 ** -53

    def random(self):
        return self._u()

    def randint(self, a, b):
        u = self._u()
        return a + math.floor(u * (b - a)) if b > a else a

    def uniform(self, a, b):
        return a + self._u() * (b - a)

    def choice_range(self, a, b):
        return self.randint(a, b)

    def choice(self, cands):
        return cands[self.randint(0, len(cands))]

    def windows(self, n, k):
        """Selection sampling (Knuth's algorithm S): window i is taken when (n - i) u < (windows still needed)."""
        sel, need = [], k
        for i in range(n):
            if need == 0:
                break
            if (n - i) * self._u() < need:
                sel.append(i)
                need -= 1
        return sel

    def normal(self, kind, chans, start, stop):
        c = np.asarray(list(chans), np.uint64)[:, None]
        i = np.arange(start, stop, dtype=np.uint64)[None, :]
        return counter_normal(self.seed, STREAM_NORMAL + kind, normal_index(self.n, self.C, c, i))


# ---- the pipeline --------------------------------------------------------------------------------------------------
class Preprocessor:
    """`DataPreprocessor` (training/preprocess.py:52-134) for `process` and the metric targets; same keyword names."""

    def __init__(self, data_channels, sampling_rate, in_samples, min_snr, p_position_ratio, coda_ratio, norm_mode,
                 add_event_rate, add_noise_rate, add_gap_rate, drop_channel_rate, scale_amplitude_rate, pre_emphasis_rate,
                 pre_emphasis_ratio, max_event_num, generate_noise_rate, shift_event_rate, mask_percent, noise_percent,
                 min_event_gap_sec, soft_label_shape="gaussian", soft_label_width=25, dtype=np.float32):
        self.data_channels, self.sampling_rate, self.in_samples = data_channels, sampling_rate, in_samples
        self.coda_ratio, self.norm_mode, self.min_snr, self.p_position_ratio = coda_ratio, norm_mode, min_snr, p_position_ratio
        self.add_event_rate, self.add_noise_rate, self.add_gap_rate = add_event_rate, add_noise_rate, add_gap_rate
        self.drop_channel_rate, self.scale_amplitude_rate = drop_channel_rate, scale_amplitude_rate
        self.pre_emphasis_rate, self.pre_emphasis_ratio = pre_emphasis_rate, pre_emphasis_ratio
        self.max_event_num, self.generate_noise_rate, self.shift_event_rate = max_event_num, generate_noise_rate, shift_event_rate
        self.mask_percent, self.noise_percent = mask_percent, noise_percent
        self.min_event_gap = int(min_event_gap_sec * sampling_rate)                              # :111
        if 0 <= p_position_ratio <= 1:                                                           # :113-130
            self.add_event_rate = self.shift_event_rate = self.generate_noise_rate = 0.0
        self.soft_label_shape, self.soft_label_width = soft_label_shape, soft_label_width
        self.log = None            # set to a dict to record the branches taken and the quantities drawn

    def _rec(self, key, value=True):
        if self.log is not None:
            self.log.setdefault(key, []).append(value)

    def is_noise(self, data, ppks, spks, snr) -> bool:                                           # :154-170
        noise = (len(ppks) != len(spks) or len(ppks) < 1 or len(spks) < 1 or min(ppks + spks) < 0
                 or max(ppks + spks) >= data.shape[-1] or (snr is not None and all(np.asarray(snr) < self.min_snr)))
        for i in range(min(len(ppks), len(spks))):       # the reference raises IndexError for more P than S picks
            noise |= ppks[i] >= spks[i]
        return bool(noise)

    def process(self, data, ppks, spks, snr, augmentation: bool, draws):
        """-> (x (C, in_samples) float32, output P list, output S list, cleared)."""
        data = np.array(data, dtype=np.float32, copy=True)
        ppks, spks = [int(v) for v in ppks], [int(v) for v in spks]
        cleared = self.is_noise(data, ppks, spks, snr)                                           # :515-521
        if cleared:
            ppks, spks = [], []
        ppks, spks = PR.pad_phases(ppks, spks, self.min_event_gap, self.in_samples)              # :523-525
        if augmentation:                                                                         # :528-529
            assert all(p >= 0 for p in ppks) and all(s < data.shape[-1] for s in spks), "padded phases reached augmentation"
            data, ppks, spks, noise = self.augment(data, ppks, spks, draws)
            cleared |= noise
        data, ppks, spks = self.cut_window(data, ppks, spks, draws)                              # :532-537
        return PR.normalize(data, self.norm_mode).astype(np.float32), ppks, spks, cleared       # :540

    def augment(self, data, ppks, spks, d):                                                      # :432-499
        noise = False
        if d.random() < self.generate_noise_rate:
            self._rec("generate_noise")
            data = self.generate_noise(data, ppks, spks, d)
            ppks, spks, noise = [], [], True
            if d.random() < self.drop_channel_rate:
                data = self.adjust_amplitude(self.drop_channel(data, d))
            if d.random() < self.scale_amplitude_rate:
                data = self.scale_amplitude(data, d)
        else:
            for _ in range(self.max_event_num - len(ppks)):
                if d.random() < self.add_event_rate and ppks:
                    data, ppks, spks = self.add_event(data, ppks, spks, d)
            if d.random() < self.shift_event_rate:
                data, ppks, spks = self.shift_event(data, ppks, spks, d)
            if d.random() < self.drop_channel_rate:
                data = self.adjust_amplitude(self.drop_channel(data, d))
            if d.random() < self.scale_amplitude_rate:
                data = self.scale_amplitude(data, d)
            if d.random() < self.pre_emphasis_rate:
                self._rec("pre_emphasis")
                data = self.pre_emphasis(data)
            if d.random() < self.add_noise_rate:
                data = self.add_noise(data, d)
            if d.random() < self.add_gap_rate:
                data = self.add_gaps(data, ppks, spks, d)
        if self.mask_percent > 0:
            data = self.windows(data, self.mask_percent, d, None)
        if self.noise_percent > 0:
            data = self.windows(data, self.noise_percent, d, NOISE_WINDOW)
        return data, ppks, spks, noise

    def generate_noise(self, data, ppks, spks, d):                                               # :244-263
        for ppk, spk in zip(ppks, spks):
            coda_end = np.clip(int(spk + self.coda_ratio * (spk - ppk)), 0, data.shape[-1], dtype=int)
            if ppk < coda_end:
                data[:, ppk:coda_end] = d.normal(NOISE_FILL, range(data.shape[0]), ppk, coda_end)
        return data

    def add_event(self, data, ppks, spks, d):                                                    # :265-292
        t = d.randint(0, len(ppks))
        ppk, spk = ppks[t], spks[t]
        coda_end = int(spk + (self.coda_ratio * (spk - ppk)))
        left = coda_end + self.min_event_gap
        right = data.shape[-1] - (spk - ppk) - self.min_event_gap
        if left < right:
            ppk_add = d.randint(left, right)
            spk_add = ppk_add + spk - ppk
            space = min(data.shape[-1] - ppk_add, coda_end - ppk)
            scale = d.random()
            self._rec("add_event", (ppk_add, scale))
            data[:, ppk_add:ppk_add + space] += data[:, ppk:ppk + space] * scale
            ppks.append(ppk_add)
            spks.append(spk_add)
        ppks.sort()
        spks.sort()
        return data, ppks, spks

    def shift_event(self, data, ppks, spks, d):                                                  # :294-305
        shift = d.randint(0, data.shape[-1])
        self._rec("shift", shift)
        data = np.concatenate((data[:, -shift:], data[:, :-shift]), axis=1)
        ppks = sorted((p + shift) % data.shape[-1] for p in ppks)
        spks = sorted((s + shift) % data.shape[-1] for s in spks)
        return data, ppks, spks

    def drop_channel(self, data, d):                                                             # :307-321
        self._rec("drop_channel")
        if data.shape[0] < 2:
            return data
        drop_num = d.choice_range(1, data.shape[0])
        candidates = list(range(data.shape[0]))
        for _ in range(drop_num):
            c = d.choice(candidates)
            candidates.remove(c)
            data[c, :] = 0.0
        return data

    def adjust_amplitude(self, data):                                                            # :323-333
        max_amp = np.max(np.abs(data), axis=1)
        if np.count_nonzero(max_amp) > 0:
            data *= data.shape[0] / np.count_nonzero(max_amp)
        return data

    def scale_amplitude(self, data, d):                                                          # :335-344
        if d.uniform(0, 1) < 0.5:
            s = d.uniform(1, 3)
            data *= s
        else:
            s = d.uniform(1, 3)
            data /= s
        self._rec("scale", s)
        return data

    def pre_emphasis(self, data):                                                                # :346-353
        for c in range(data.shape[0]):
            bpf = data[c, :]
            data[c, :] = np.append(bpf[0], bpf[1:] - self.pre_emphasis_ratio * bpf[:-1])
        return data

    def add_noise(self, data, d):                                                                # :355-368
        for c in range(data.shape[0]):
            x = data[c, :]
            snr = d.randint(10, 50)
            self._rec("snr", snr)
            px = np.sum(x ** 2) / len(x)
            pn = px * 10 ** (-snr / 10.0)
            noise = d.normal(NOISE_ADD, [c], 0, len(x))[0] * np.sqrt(pn)
            data[c, :] += noise
        return data

    def add_gaps(self, data, ppks, spks, d):                                                     # :370-390
        phases = sorted(ppks + spks)
        if len(phases) > 0:
            phases.append(data.shape[-1] - 1)
            phases = sorted(set(phases))
            insert_pos = d.randint(0, len(phases) - 1)
            sgt = d.randint(phases[insert_pos], phases[insert_pos + 1])
            egt = d.randint(sgt, phases[insert_pos + 1])
            self._rec("gap", (sgt, egt, phases[insert_pos], phases[insert_pos + 1]))
        else:
            sgt = d.randint(0, data.shape[-1] - 1)
            egt = d.randint(sgt + 1, data.shape[-1])
            self._rec("gap", (sgt, egt, 0, data.shape[-1]))
        data[:, sgt:egt] = 0
        return data

    def windows(self, data, percent, d, kind):                                                   # :392-430
        window_size = self.sampling_rate // 2
        p = np.clip(percent, 0, 100)
        num_windows = data.shape[-1] // window_size
        for i in d.windows(num_windows, num_windows * p // 100):
            st, et = i * window_size, i * window_size + window_size
            data[:, st:et] = 1.0 if kind is None else d.normal(kind, range(data.shape[0]), st, et)
        return data

    def cut_window(self, data, ppks, spks, d):                                                   # :172-222
        input_len, window_size = data.shape[-1], self.in_samples
        if 0 <= self.p_position_ratio <= 1:
            new_data = np.zeros((data.shape[0], window_size), dtype=np.float32)
            tgt_l, tgt_r = 0, window_size
            # the reference raises IndexError for an event without P: the device cuts it from sample 0
            p_idx = ppks[0] if ppks else int(window_size * self.p_position_ratio)
            c_l = p_idx - int(window_size * self.p_position_ratio)
            c_r = c_l + window_size
            offset = -c_l
            if c_l < 0:
                tgt_l += abs(c_l)
                offset += c_l
                c_l = 0
            if c_r > data.shape[-1]:
                tgt_r -= c_r - data.shape[-1]
                c_r = data.shape[-1]
            new_data[:, tgt_l:tgt_r] = data[:, c_l:c_r]
            offset += tgt_l
            data = new_data
            ppks = [t + offset for t in ppks if 0 <= t + offset < window_size]
            spks = [t + offset for t in spks if 0 <= t + offset < window_size]
        elif input_len > window_size:
            c_l = d.randint(0, max(min(ppks + [input_len - window_size]) - self.min_event_gap, 1))
            self._rec("cut", (c_l, max(min(ppks + [input_len - window_size]) - self.min_event_gap, 1)))
            c_r = c_l + window_size
            data = data[:, c_l:c_r]
            ppks = [t - c_l for t in ppks if c_l <= t < c_r]
            spks = [t - c_l for t in spks if c_l <= t < c_r]
        elif input_len < window_size:
            data = np.concatenate([data, np.zeros((data.shape[0], window_size - input_len))], axis=1)   # float64
        return data, ppks, spks

    # ---- get_targets_for_metrics :761-804 for det / ppk / spk ----------------------------------------------------------
    def expected_det_num(self) -> int:
        return (self.max_event_num + int(bool(self.add_event_rate)) + int(bool(self.shift_event_rate))
                + int(0 <= self.p_position_ratio <= 1))

    def metric_targets(self, ppks, spks):
        """{"ppk", "spk": phase lists padded with int(-1e7) to max_event_num, "det": [st, et, ...] padded with [1, 0]}.
        A list longer than max_event_num raises, as `_pad_array` does."""
        out = {}
        for name, ph in (("ppk", ppks), ("spk", spks)):
            v = np.array(ph).astype(np.float32)
            if len(v) > self.max_event_num:
                raise ValueError(f"`length < len(s)` . Array:{len(v)},Target:{self.max_event_num}")
            out[name] = np.pad(v, (0, self.max_event_num - len(v)), mode="constant", constant_values=int(-1e7)).astype(np.int64)
        pp, ss = PR.pad_phases(ppks, spks, self.soft_label_width, self.in_samples)
        det = []
        for ppk, spk in zip(pp, ss):
            det.extend([np.clip(ppk, 0, self.in_samples), int(spk + (self.coda_ratio * (spk - ppk)))])
        if len(det) // 2 < self.expected_det_num():
            det = det + [1, 0] * (self.expected_det_num() - len(det) // 2)
        out["det"] = np.array(det).astype(np.int64)
        return out


# ---- soft labels with the sigmoid window -----------------------------------------------------------------------------
def window(width: int, shape: str) -> np.ndarray:
    """oracle/preprocess_ref.py::window plus the sigmoid shape (:586-597)."""
    if shape != "sigmoid":
        return PR.window(width, shape)
    left = int(width / 2)
    right = width - left
    l_l, l_r = -int(left / 2), left - int(left / 2)
    r_l, r_r = -int(right / 2), right - int(right / 2)
    x_l, x_r = -10 / left * np.arange(l_l, l_r), -10 / right * (-1) * np.arange(r_l, r_r)
    return np.concatenate((1 / (1 + np.exp(x_l)), [1.0], 1 / (1 + np.exp(x_r))), axis=0)


def soft_label(idxs, length: int, width: int, shape: str) -> np.ndarray:
    lab = np.zeros(length)
    left = int(width / 2)
    w = window(width, shape)
    for idx in idxs:
        if idx < 0 or idx > length - 1:
            continue
        lo, hi = idx - left, idx - left + len(w)
        a, b = max(lo, 0), min(hi, length)
        lab[a:b] += w[a - lo:b - lo]
    return lab


def dpk_labels(ppks, spks, length: int, width: int, shape: str, coda_ratio: float) -> np.ndarray:
    """oracle/preprocess_ref.py::dpk_labels for every shape, sigmoid included."""
    pp, ss = PR.pad_phases(ppks, spks, width, length)
    det = np.zeros(length)
    clip = lambda v: min(max(v, 0), length)      # noqa: E731
    for ppk, spk in zip(pp, ss):
        e = int(spk + coda_ratio * (spk - ppk))
        li = soft_label([ppk, e], length, width, shape)
        li[clip(ppk):clip(e)] = 1.0
        det += li
    det[det > 1] = 1.0
    return np.stack([det, soft_label(ppks, length, width, shape), soft_label(spks, length, width, shape)]).astype(np.float32)
