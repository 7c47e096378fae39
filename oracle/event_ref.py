"""CPU oracle (TEST INFRASTRUCTURE) of the P-anchored event window (seist_b200/events.py, DESIGN §4.17), restated in numpy
from the reference's training/preprocess.py: `DataPreprocessor._cut_window` with 0 <= p_position_ratio <= 1 (:172-203)
then `_normalize` (:224-242), in float32 exactly as numpy executes the reference (float32 window, numpy's float32 mean and
std), so it equals tests/golden/reference_event_windows.pt bit for bit.

For a pick outside [0, T) the reference's slices wrap around through negative indices; the device gives a zero row there
and so does `window` (the picker never produces such picks).
"""
import numpy as np

from oracle.preprocess_ref import normalize


def anchor(window: int, p_position_ratio: float) -> int:
    """`int(window_size * self.p_position_ratio)`: the sample of the window that holds the P pick."""
    return int(window * p_position_ratio)


def cut(trace: np.ndarray, p: int, window: int, a: int) -> np.ndarray:
    """(C, window) float32: trace[:, p - a + i] for i < window, zero where p - a + i falls outside [0, T)."""
    C, T = trace.shape
    out = np.zeros((C, window), dtype=np.float32)
    if not 0 <= p < T:
        return out
    lo, hi = max(p - a, 0), min(p - a + window, T)
    if lo < hi:
        out[:, lo - (p - a):hi - (p - a)] = trace[:, lo:hi]
    return out


def window(trace: np.ndarray, p: int, window_size: int, p_position_ratio: float, mode: str) -> np.ndarray:
    """The model input of the event whose first P pick is p on trace (C, T)."""
    return normalize(cut(trace, p, window_size, anchor(window_size, p_position_ratio)), mode)


def windows(record: np.ndarray, index: np.ndarray, offsets: np.ndarray, window_size: int, p_position_ratio: float,
            mode: str) -> np.ndarray:
    """(M, C, window) for every pick of the CSR (index (M,), offsets (S + 1,)) on record (S, C, T)."""
    C = record.shape[1]
    out = np.zeros((len(index), C, window_size), dtype=np.float32)
    for s in range(record.shape[0]):
        for e in range(int(offsets[s]), int(offsets[s + 1])):
            out[e] = window(record[s], int(index[e]), window_size, p_position_ratio, mode)
    return out
