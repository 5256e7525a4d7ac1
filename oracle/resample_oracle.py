"""Float64 numpy restatement of the resampling the reference's preprocessing runs (DESIGN.md section 22): its
`read_wav_np` calls `librosa.load(path, sr=...)` for a file at another rate, and librosa 0.7.0 (the pinned version)
resamples with resampy 0.2.x, `res_type='kaiser_best'`, then `fix_length`s the result to ceil(N * ratio) samples.

Neither library is needed here: equality with them holds by construction, not by test.  This module restates resampy's
`resample_f` loop in its own operation order (every product and sum rounded on its own, the output rounded to float32
after every tap because resampy accumulates into a float32 array), and the GPU kernel (csrc/resample.cu) matches it
bit for bit.  resampy ships its Kaiser-windowed sinc table as a data file; `filter_table` rebuilds it with resampy's
`sinc_window` recipe, and whether current numpy / scipy reproduce that file bit for bit is unverified.

The loop is vectorised over output samples, one tap index at a time, so each output's taps are still summed in
resampy's order (left wing i = 0, 1, ..., then right wing k = 0, 1, ...).  The time register is np.add.accumulate,
which adds sequentially, as resampy's running `time_register += time_increment` does."""
from __future__ import annotations

import numpy as np
import scipy.signal

NUM_ZEROS = 64
PRECISION = 9
NUM_TABLE = 1 << PRECISION                     # 512 table entries per zero crossing
N_WIN = NUM_TABLE * NUM_ZEROS + 1              # 32769: the right wing, both ends included
ROLLOFF = 0.9475937167399596
BETA = 14.769656459379492


def filter_table(sr_orig: int, sr_new: int):
    """(win, delta), float64 [N_WIN] each: resampy's kaiser_best right wing, scaled by the ratio when downsampling, and
    its forward difference (delta[-1] = 0) taken after the scaling."""
    n = NUM_TABLE * NUM_ZEROS
    sinc = ROLLOFF * np.sinc(ROLLOFF * np.linspace(0, NUM_ZEROS, num=n + 1, endpoint=True))
    win = scipy.signal.windows.kaiser(2 * n + 1, BETA)[n:] * sinc
    ratio = float(sr_new) / sr_orig
    if ratio < 1:
        win = win * ratio
    delta = np.zeros_like(win)
    delta[:-1] = np.diff(win)
    return win, delta


def out_lengths(N: int, sr_orig: int, sr_new: int):
    """(n_out, M): the samples resampy computes, int(N * ratio), and the length librosa fixes them to, ceil(N * ratio)."""
    r = float(sr_new) / sr_orig
    return int(N * r), int(np.ceil(N * r))


def resample(x, sr_orig: int, sr_new: int, table=None) -> np.ndarray:
    """x float32 [N] at sr_orig -> float32 [ceil(N * ratio)] at sr_new (librosa.resample(x, sr_orig, sr_new) with
    res_type='kaiser_best', fix_length included).  sr_orig == sr_new returns x.  Raises ValueError when
    int(N * ratio) < 1, as resampy does."""
    x = np.asarray(x, dtype=np.float32)
    if sr_orig == sr_new:
        return x
    N = x.shape[0]
    n_out, M = out_lengths(N, sr_orig, sr_new)
    if n_out < 1:
        raise ValueError(f"input of {N} samples is too short to resample from {sr_orig} to {sr_new} Hz")
    win, delta = table if table is not None else filter_table(sr_orig, sr_new)
    ratio = float(sr_new) / sr_orig
    scale = min(1.0, ratio)
    step = int(scale * NUM_TABLE)
    reg = np.add.accumulate(np.concatenate([[0.0], np.full(n_out - 1, 1.0 / ratio)]))
    n = reg.astype(np.int64)
    x64 = x.astype(np.float64)
    y = np.zeros(n_out, dtype=np.float32)
    frac = scale * (reg - n)
    for wing, f in ((0, frac), (1, scale - frac)):
        index_frac = f * NUM_TABLE
        offset = index_frac.astype(np.int64)
        eta = index_frac - offset
        lim = (N_WIN - offset) // step
        count = np.minimum(n + 1, lim) if wing == 0 else np.minimum(N - n - 1, lim)
        for i in range(int(count.max(initial=0))):
            m = np.nonzero(i < count)[0]
            j = offset[m] + i * step
            w = win[j] + eta[m] * delta[j]
            src = n[m] - i if wing == 0 else n[m] + i + 1
            y[m] = (y[m].astype(np.float64) + w * x64[src]).astype(np.float32)
    out = np.zeros(M, dtype=np.float32)
    out[:n_out] = y
    return out


def backend(wavs, sr_orig: int, sr_new: int):
    """The preprocessing command's resampling hook on the oracle: a list of float32 wavs at sr_orig -> the list at sr_new."""
    table = filter_table(sr_orig, sr_new)
    return [resample(w, sr_orig, sr_new, table) for w in wavs]
