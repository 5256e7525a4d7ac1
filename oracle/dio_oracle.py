"""CPU restatement of the reference's feature extraction (nvidia_preprocessing.py, compute_statistics.py), the contract of
`fastspeech2_b200.features` (DESIGN.md section 14).  TEST INFRASTRUCTURE ONLY.

  mel, energy   `oracle.stft_oracle.STFT` + the package's librosa-0.7 mel filterbank + log(clamp(., 1e-5)): what
                `TacotronSTFT.mel_spectrogram` computes (utils/stft.py:188-204), and torch.norm(|STFT|, dim=0)
  pitch         WORLD's DIO as pyworld 0.2.10 runs it with the reference's defaults (dataset/audio_processing.py:54-70),
                restated in float64 numpy from the published algorithm (Morise, Kawahara and Katayose 2009; the WORLD
                vocoder's dio.cpp), with np.fft for the filters like WORLD.  pyworld itself is not available to this
                project, so equality with `pyworld.dio` is by construction, not by test.

DIO, step by step (DESIGN.md section 14 lists the same):
  1. bands      n_bands = 1 + int(log2(f0_ceil / f0_floor) * channels_in_octave); boundary[i] = f0_floor * 2^((i+1) / cio).
                speed = 1: no decimation; y_length = N + 1; fft_size = the smallest power of two > y_length +
                4 * int(1 + fs / boundary[0] / 2).
  2. DC         y = x, then one zero; subtract the mean of y[0:y_length] (so y[N] = -mean).
  3. low cut    zero-phase circular FIR of N_lc = 2 * round(fs / 50) + 1 taps: delta minus the normalised Hann
                0.5 - 0.5 cos(2 pi i / (N_lc + 1)), i = 1..N_lc, centred on index 0 modulo fft_size.
  4. bands      per band, h = round(fs / boundary / 2): a 4h-tap Nuttall window (0.355768, 0.487396, 0.144232, 0.012604)
                as a circular FIR, advanced by 2h samples; s = filtered[0:y_length].
  5. events     four series: negative-going zero crossings of s (0 < g[i] and g[i+1] <= 0, edge e = i + 1), of -s, of
                the difference of -s (d[i] = (-s[i]) - (-s[i+1]), over y_length - 1 samples: peaks of s) and of -d
                (dips).  fine edge e - g[e-1] / (g[e] - g[e-1]); each consecutive pair gives fs / delta at (mid) / fs.
                A series with fewer than 3 intervals makes the band's candidate 0 with score 1e5 on every frame.
  6. candidates interp1 / histc (linear, extrapolating from the end segments) at t_i = i * frame_period / 1000; mean of
                the four, score = their standard deviation with divisor 3; 0 / 1e5 outside
                [max(boundary / 2, f0_floor), min(boundary, f0_ceil)]; score /= candidate + 1e-12.
  7. best band  band 0, then band j where its score is strictly smaller (the first minimum wins).
  8. FixF0Contour, with vrm = int(0.5 + 1000 / frame_period / f0_floor) * 2 + 1 (all zeros if f0_length <= vrm):
                step 1 zeroes the first and last vrm frames and jumps |(f[i] - f[i-1]) / (1e-12 + f[i])| >= allowed_range;
                step 2 zeroes frames with a zero within +-(vrm - 1) / 2; step 3 extends each voiced section forward
                from its last frame with SelectBestF0 (reference (3 f[j] - f[j-1]) / 2, nearest candidate over all
                bands, rejected when |1 - best / ref| > allowed_range), up to the next section's last frame (the last
                frame for the last section) or the first rejection; step 4 does the same backwards from each section's
                first frame, last section first, down to the previous section's first frame (frame 1 for the first).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle.stft_oracle import STFT

K_LOG2 = 0.69314718055994529          # WORLD's kLog2
K_MAX = 100000.0                       # kMaximumValue
K_SAFE = 1e-12                         # kMySafeGuardMinimum


def matlab_round(x: float) -> int:
    return int(x + 0.5) if x > 0 else int(x - 0.5)


def frame_period_ms(hop: int, fs: int) -> float:
    """The reference's `frame_period=hop / fs * 1000`."""
    return hop / fs * 1000


def f0_length(n: int, fs: int, frame_period: float) -> int:
    """WORLD's GetSamplesForDIO, evaluated in double in the same order."""
    return int(1000.0 * n / fs / frame_period) + 1


def band_edges(f0_floor=71.0, f0_ceil=800.0, channels_in_octave=2.0) -> np.ndarray:
    n_bands = 1 + int(math.log(f0_ceil / f0_floor) / K_LOG2 * channels_in_octave)
    return np.array([f0_floor * 2.0 ** ((i + 1) / channels_in_octave) for i in range(n_bands)])


def fft_size(n: int, fs: int, boundary0: float) -> int:
    """Smallest power of two strictly greater than y_length + 4 * int(1 + fs / boundary0 / 2)."""
    m = n + 1 + 4 * int(1.0 + fs / boundary0 / 2.0)
    return 1 << m.bit_length()


def lowcut_taps(fs: int) -> np.ndarray:
    """The low-cut filter's taps at offsets -M..M (M = round(fs / 50)), delta included: DesignLowCutFilter.  The Hann
    normaliser is summed in order, like WORLD's loop."""
    n = matlab_round(fs / 50.0) * 2 + 1
    w = 0.5 - 0.5 * np.cos(np.arange(1, n + 1) * 2.0 * np.pi / (n + 1))
    total = 0.0
    for v in w:
        total += v
    taps = -w / total
    taps[(n - 1) // 2] += 1.0
    return taps


def nuttall(n: int) -> np.ndarray:
    t = np.arange(n) / (n - 1.0)
    return 0.355768 - 0.487396 * np.cos(2.0 * np.pi * t) + 0.144232 * np.cos(4.0 * np.pi * t) - 0.012604 * np.cos(6.0 * np.pi * t)


def _fine_edges(g: np.ndarray) -> np.ndarray:
    e = np.nonzero((g[:-1] > 0.0) & (g[1:] <= 0.0))[0] + 1
    return e - g[e - 1] / (g[e] - g[e - 1])


def _series(fine: np.ndarray, fs: float):
    """(locations, intervals) of consecutive edge pairs; empty when there are fewer than two edges."""
    if len(fine) < 2:
        return np.zeros(0), np.zeros(0)
    return (fine[:-1] + fine[1:]) / 2.0 / fs, fs / (fine[1:] - fine[:-1])


def interp1(x: np.ndarray, y: np.ndarray, xi: np.ndarray) -> np.ndarray:
    """WORLD's interp1 with histc: segment k = min(1 + #{j >= 1: x[j] <= xi}, len(x) - 1), extrapolating at both ends."""
    k = np.minimum(1 + np.searchsorted(x[1:], xi, side="right"), len(x) - 1)
    s = (xi - x[k - 1]) / (x[k] - x[k - 1])
    return y[k - 1] + s * (y[k] - y[k - 1])


def _select_best(cur, past, cands, idx, allowed):
    ref = (cur * 3.0 - past) / 2.0
    best, err = cands[0, idx], abs(ref - cands[0, idx])
    for j in range(1, cands.shape[0]):
        e = abs(ref - cands[j, idx])
        if e < err:
            err, best = e, cands[j, idx]
    return 0.0 if abs(1.0 - best / ref) > allowed else best


def fix_f0_contour(best: np.ndarray, cands: np.ndarray, frame_period: float, f0_floor: float, allowed: float) -> np.ndarray:
    n = len(best)
    vrm = int(0.5 + 1000.0 / frame_period / f0_floor) * 2 + 1
    out = np.zeros(n)
    if n <= vrm:
        return out
    base = best.copy()
    base[:vrm] = 0.0
    base[n - vrm:] = 0.0
    s1 = np.zeros(n)
    for i in range(vrm, n):
        s1[i] = base[i] if abs((base[i] - base[i - 1]) / (K_SAFE + base[i])) < allowed else 0.0
    s2 = s1.copy()
    c = (vrm - 1) // 2
    for i in range(c, n - c):
        if np.any(s1[i - c: i + c + 1] == 0):
            s2[i] = 0.0
    neg, pos = [], []
    for i in range(1, n):
        if s2[i] == 0 and s2[i - 1] != 0:
            neg.append(i - 1)
        elif s2[i - 1] == 0 and s2[i] != 0:
            pos.append(i)
    f = s2.copy()
    for i, start in enumerate(neg):                                   # step 3
        limit = n - 1 if i == len(neg) - 1 else neg[i + 1]
        for j in range(start, limit):
            f[j + 1] = _select_best(f[j], f[j - 1], cands, j + 1, allowed)
            if f[j + 1] == 0:
                break
    for i in range(len(pos) - 1, -1, -1):                             # step 4
        limit = 1 if i == 0 else pos[i - 1]
        for j in range(pos[i], limit, -1):
            f[j - 1] = _select_best(f[j], f[j + 1], cands, j - 1, allowed)
            if f[j - 1] == 0:
                break
    return f


def dio(x, fs: int, f0_floor=71.0, f0_ceil=800.0, channels_in_octave=2.0, frame_period=5.0, allowed_range=0.1,
        return_bands=False):
    """float64 f0 contour of length f0_length(len(x), fs, frame_period) (what `pyworld.dio(x, fs, ...)[0]` returns)."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    boundary = band_edges(f0_floor, f0_ceil, channels_in_octave)
    y_length = n + 1
    F = fft_size(n, fs, boundary[0])
    y = np.zeros(F)
    y[:n] = x
    y[:y_length] -= y[:y_length].sum() / y_length
    lc = lowcut_taps(fs)
    m = (len(lc) - 1) // 2
    lc_c = np.zeros(F)
    lc_c[np.arange(-m, m + 1) % F] = lc                               # centred on 0, wrapped like WORLD's layout
    spec = np.fft.rfft(y) * np.fft.rfft(lc_c)
    T = f0_length(n, fs, frame_period)
    ti = np.arange(T) * frame_period / 1000.0
    cands = np.zeros((len(boundary), T))
    scores = np.zeros((len(boundary), T))
    for j, b in enumerate(boundary):
        h = matlab_round(fs / b / 2.0)
        nut = np.zeros(F)
        nut[: 4 * h] = nuttall(4 * h)
        filt = np.fft.irfft(spec * np.fft.rfft(nut), F)
        s = filt[2 * h: 2 * h + y_length]
        d = (-s[:-1]) - (-s[1:])
        series = [_series(_fine_edges(g), float(fs)) for g in (s, -s, d, -d)]
        if min(len(loc) for loc, _ in series) < 3:
            c, sc = np.zeros(T), np.full(T, K_MAX)
        else:
            v = [interp1(loc, iv, ti) for loc, iv in series]
            c = (v[0] + v[1] + v[2] + v[3]) / 4.0
            sc = np.sqrt(((v[0] - c) * (v[0] - c) + (v[1] - c) * (v[1] - c) + (v[2] - c) * (v[2] - c) + (v[3] - c) * (v[3] - c)) / 3.0)
            bad = (c > b) | (c < b / 2.0) | (c > f0_ceil) | (c < f0_floor)
            c = np.where(bad, 0.0, c)
            sc = np.where(bad, K_MAX, sc)
        cands[j], scores[j] = c, sc / (c + K_SAFE)
    best = cands[0].copy()
    bs = scores[0].copy()
    for j in range(1, len(boundary)):
        upd = bs > scores[j]
        bs = np.where(upd, scores[j], bs)
        best = np.where(upd, cands[j], best)
    f0 = fix_f0_contour(best, cands, frame_period, f0_floor, allowed_range)
    return (f0, cands, best) if return_bands else f0


def mel_energy(x, sample_rate=22050, n_fft=1024, hop=256, win_length=1024, n_mels=80, fmin=0.0, fmax=8000.0):
    """(mel [n_mels, T] float32, energy [T] float32), T = len(x) // hop + 1: TacotronSTFT.mel_spectrogram's log-mel and
    nvidia_preprocessing.py's torch.norm(mag, dim=0)."""
    from fastspeech2_b200.vocoder import mel_filterbank
    st = STFT(n_fft, hop, win_length)
    mag, _ = st.transform(torch.as_tensor(np.asarray(x, dtype=np.float32))[None])
    basis = torch.from_numpy(mel_filterbank(sample_rate, n_fft, n_mels, fmin, fmax))
    mel = torch.log(torch.clamp(torch.matmul(basis, mag[0]), min=1e-5))
    return mel.numpy(), torch.norm(mag[0], dim=0).numpy()


def features(x, sample_rate=22050, n_fft=1024, hop=256, win_length=1024, n_mels=80, fmin=0.0, fmax=8000.0,
             f0_floor=71.0, f0_ceil=800.0, channels_in_octave=2.0, allowed_range=0.1):
    """What nvidia_preprocessing.py writes for one utterance: (mel [n_mels, T] float32, energy [T] float32,
    pitch [min(f0_length, T)] float64)."""
    mel, e = mel_energy(x, sample_rate, n_fft, hop, win_length, n_mels, fmin, fmax)
    p = dio(np.asarray(x, dtype=np.float32).astype(np.float64), sample_rate, f0_floor, f0_ceil, channels_in_octave,
            frame_period_ms(hop, sample_rate), allowed_range)
    return mel, e, p[: mel.shape[1]]

