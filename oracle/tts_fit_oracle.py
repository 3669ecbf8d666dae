"""Float32 NumPy statement of the duration-fit rule (include/ovc.h: ovc_tts_fit; openvoice_b200/csrc/ovc_tts_ops.h).

A fit group of rows with logw [R, T] and token counts lens [R] has, at an fp32 length scale s,
F(s) = sum_r max(1, sum_{t < len_r} ceil(float32(exp(logw_r[t])) * s)) frames: the y_lengths of
``SynthesizerTrn.infer(..., length_scale=s)`` (openvoice/models.py:477-479).  Its fitted scale is the smallest fp32 s
in [lo, hi] with F(s) >= target, or hi when there is none.  Everything is float32 as in the reference, and the frames
add up in int64."""
from __future__ import annotations

import numpy as np

SCALE_LO, SCALE_HI = 0.25, 4.0


def bits(s) -> int:
    return int(np.array(s, np.float32).view(np.uint32))


def from_bits(u: int) -> np.float32:
    return np.array(u, np.uint32).view(np.float32)[()]


def token_frames(e: np.ndarray, s) -> np.ndarray:
    """ceil(e * s) in float32 as int64; a NaN or a count past 2^30 saturates at 2^30."""
    w = np.ceil(e.astype(np.float32) * np.float32(s))
    return np.where(w < 2.0 ** 30, w, 2.0 ** 30).astype(np.int64)


def group_frames(e: np.ndarray, lens: np.ndarray, s) -> int:
    """F(s) of the rows of e = float32 exp(logw) [R, T] with token counts lens [R]."""
    e = np.asarray(e, np.float32).reshape(len(lens), -1)
    mask = np.arange(e.shape[1])[None, :] < np.clip(np.asarray(lens), 0, e.shape[1])[:, None]
    n = np.where(mask, token_frames(e, s), 0).sum(1)
    return int(np.maximum(n, 1).sum())


def fit_scale(e: np.ndarray, lens: np.ndarray, target: int, lo=SCALE_LO, hi=SCALE_HI) -> np.float32:
    """The fitted scale: bisection over the ordered bit patterns of the floats in [lo, hi]."""
    a, b = bits(lo), bits(hi)
    while a < b:
        mid = a + (b - a) // 2
        if group_frames(e, lens, from_bits(mid)) >= target:
            b = mid
        else:
            a = mid + 1
    return from_bits(a)


def fit_scale_logw(logw: np.ndarray, lens: np.ndarray, target: int, lo=SCALE_LO, hi=SCALE_HI) -> np.float32:
    return fit_scale(np.exp(np.asarray(logw, np.float32)), lens, target, lo, hi)
