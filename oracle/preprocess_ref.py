"""CPU oracle (TEST INFRASTRUCTURE) for the input side of SURVEY §8f-3: per-trace normalisation and the soft labels of
the dpk task, restated in numpy from the reference's training/preprocess.py:

  * `normalize`        — `DataPreprocessor._normalize` :224-242 (mean removal per channel, then max or std scaling;
                         note: `max` is the signed maximum, not max |x|, and a zero scale is replaced by 1);
  * `soft_label`       — `_get_soft_label` inside `_generate_soft_label` :565-615 (gaussian exp(-d^2/200) / triangle / box
                         windows of `width + 1` samples added at every phase index, clipped at the trace borders);
  * `det_label`        — the `det` branch :643-656 (box from P to S + coda_ratio * (S - P) with window shoulders, <= 1);
  * `dpk_labels`       — the label stack [det, ppk, spk] of config.py:137-146 after `_pad_phases` :16-35.
Pinned in tests/test_cpu_preprocess.py by executing the reference's own method sources (extracted with `ast`; the module
itself imports h5py-backed datasets and does not import here).
"""
import numpy as np


def normalize(data: np.ndarray, mode: str) -> np.ndarray:
    data = np.array(data, copy=True)
    data -= np.mean(data, axis=1, keepdims=True)
    if mode == "max":
        m = np.max(data, axis=1, keepdims=True)
        m[m == 0] = 1
        data /= m
    elif mode == "std":
        s = np.std(data, axis=1, keepdims=True)
        s[s == 0] = 1
        data /= s
    elif mode != "":
        raise ValueError(f"Supported mode: 'max','std', got '{mode}'")
    return data


def window(width: int, shape: str) -> np.ndarray:
    left = int(width / 2)
    right = width - left
    d = np.arange(-left, right + 1)
    if shape == "gaussian":
        return np.exp(-(d ** 2) / (2 * 10 ** 2))
    if shape == "triangle":
        return 1 - np.abs(2 / width * d)
    if shape == "box":
        return np.ones(width + 1)
    raise NotImplementedError(shape)


def soft_label(idxs, length: int, width: int, shape: str) -> np.ndarray:
    lab = np.zeros(length)
    left = int(width / 2)
    w = window(width, shape)
    for idx in idxs:
        if idx < 0 or idx > length - 1:
            continue
        lo, hi = idx - left, idx - left + len(w)          # window covers [lo, hi)
        a, b = max(lo, 0), min(hi, length)
        lab[a:b] += w[a - lo:b - lo]
    return lab


def pad_phases(ppks, spks, padding_idx: int, num_samples: int):
    """_pad_phases :16-35"""
    padding_idx = abs(padding_idx)
    ppks, spks = sorted(ppks), sorted(spks)
    p, s = np.array(ppks), np.array(spks)
    i = 0
    while i < min(len(ppks), len(spks)) and all(p[: i + 1] < s[-i - 1:]):
        i += 1
    return len(s[: len(s) - i]) * [-padding_idx] + ppks, spks + len(p[i:]) * [num_samples + padding_idx]


def det_label(ppks, spks, length: int, width: int, shape: str, coda_ratio: float) -> np.ndarray:
    lab = np.zeros(length)
    clip = lambda v: min(max(v, 0), length)      # noqa: E731
    for ppk, spk in zip(ppks, spks):
        det = int(spk + coda_ratio * (spk - ppk))
        li = soft_label([ppk, det], length, width, shape)
        li[clip(ppk):clip(det)] = 1.0
        lab += li
    lab[lab > 1] = 1.0
    return lab


def dpk_labels(ppks, spks, length: int, width: int, shape: str, coda_ratio: float) -> np.ndarray:
    """(3, length) float32: det, ppk, spk for one waveform."""
    pp, ss = pad_phases(ppks, spks, width, length)
    return np.stack([det_label(pp, ss, length, width, shape, coda_ratio),
                     soft_label(ppks, length, width, shape),
                     soft_label(spks, length, width, shape)]).astype(np.float32)
