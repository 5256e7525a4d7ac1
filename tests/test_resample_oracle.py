"""The resampling oracle (oracle/resample_oracle.py) without a device: the vectorised restatement against a literal
per-sample double loop of resampy's `resample_f`, the filter table, pass- and stopband behaviour, and torchaudio's
kaiser_best emulation as a loose sanity bound.

Gates are about 4x what the oracle measures on the CPU with these inputs (1 s of signal, the middle half compared):
  DC at 48 kHz -> 22.05 kHz     |y - 0.5| <= 1e-3   (measured 2.5e-4: index_step = 235, not 235.2, so the downsampling
                                                      filter is not an exact Kaiser-sinc; 3.6e-7 at the other pairs)
  1 kHz tone, any pair          rms ratio within 2e-3 of 1    (measured 4.8e-4 at 48 kHz -> 22.05 kHz, below 1e-7 elsewhere)
  tone at 1.1x the new Nyquist  rms ratio <= 1e-3   (measured 1.9e-4 at 48 kHz -> 22.05 kHz, 1.1e-7 at 44.1 kHz)
  torchaudio sinc_interp_kaiser, width 64, same rolloff and beta, 440 Hz tone plus noise: |diff| <= 2e-3 (measured
                                                      7.1e-4 at 48 kHz -> 22.05 kHz, 3.8e-4 to 5.0e-4 elsewhere)"""
import numpy as np
import pytest
import torch

from fastspeech2_b200.resample import filter_table
from oracle import resample_oracle as R

PAIRS = [(48000, 22050), (44100, 22050), (24000, 22050), (16000, 22050), (8000, 22050), (22050, 48000), (22050, 16000)]


def literal(x, sr_orig, sr_new):
    """resampy 0.2.x resample_f, one output sample and one tap at a time, then librosa's fix_length."""
    win, delta = R.filter_table(sr_orig, sr_new)
    ratio = float(sr_new) / sr_orig
    scale, time_increment = min(1.0, ratio), 1.0 / ratio
    step = int(scale * R.NUM_TABLE)
    N, n_out = len(x), int(len(x) * ratio)
    y = np.zeros(n_out, dtype=np.float32)
    time_register = 0.0
    for t in range(n_out):
        n = int(time_register)
        frac = scale * (time_register - n)
        index_frac = frac * R.NUM_TABLE
        offset = int(index_frac)
        eta = index_frac - offset
        for i in range(min(n + 1, (R.N_WIN - offset) // step)):
            w = win[offset + i * step] + eta * delta[offset + i * step]
            y[t] = np.float32(float(y[t]) + w * float(x[n - i]))
        frac = scale - frac
        index_frac = frac * R.NUM_TABLE
        offset = int(index_frac)
        eta = index_frac - offset
        for k in range(min(N - n - 1, (R.N_WIN - offset) // step)):
            w = win[offset + k * step] + eta * delta[offset + k * step]
            y[t] = np.float32(float(y[t]) + w * float(x[n + k + 1]))
        time_register += time_increment
    out = np.zeros(int(np.ceil(N * ratio)), dtype=np.float32)
    out[:n_out] = y
    return out


def _lengths(sr_orig, sr_new):
    """1 to a few thousand samples, with the shortest accepted length and one where int(N * r) < ceil(N * r)."""
    r = float(sr_new) / sr_orig
    first = next(n for n in range(1, 100) if int(n * r) >= 1)
    ragged = next(n for n in range(first + 1, 200) if int(n * r) != int(np.ceil(n * r)))
    return sorted({1, first, ragged, 97, 640, 2501})


@pytest.mark.parametrize("sr_orig, sr_new", PAIRS)
def test_vectorised_oracle_matches_the_literal_loop(sr_orig, sr_new):
    rng = np.random.default_rng(sr_orig + sr_new)
    r = float(sr_new) / sr_orig
    for N in _lengths(sr_orig, sr_new):
        x = (0.4 * rng.standard_normal(N)).astype(np.float32)
        if int(N * r) < 1:
            with pytest.raises(ValueError, match="too short"):
                R.resample(x, sr_orig, sr_new)
            continue
        got, want = R.resample(x, sr_orig, sr_new), literal(x, sr_orig, sr_new)
        assert got.dtype == np.float32 and got.shape == (int(np.ceil(N * r)),)
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), (N, np.abs(got - want).max())
        assert not got[int(N * r):].any()


def test_shortest_inputs_are_refused_or_padded():
    assert R.out_lengths(1, 48000, 22050) == (0, 1)
    assert R.out_lengths(3, 48000, 22050) == (1, 2)
    with pytest.raises(ValueError):
        R.resample(np.ones(2, np.float32), 48000, 22050)
    assert R.resample(np.ones(3, np.float32), 48000, 22050)[1] == 0.0
    x = np.arange(5, dtype=np.float32)
    assert R.resample(x, 22050, 22050) is x


def test_filter_table_shape_and_end_values():
    win, delta = R.filter_table(22050, 48000)
    assert win.shape == delta.shape == (R.N_WIN,) == (32769,) and win.dtype == np.float64
    assert win[0] == R.ROLLOFF                          # sinc(0) = 1 under the Kaiser window's peak of 1
    assert abs(win[-1]) < 1e-7 and delta[-1] == 0.0
    assert np.array_equal(delta[:-1], np.diff(win))
    dwin, ddelta = R.filter_table(48000, 22050)         # downsampling scales the table, and delta is taken after it
    assert np.array_equal(dwin, win * (22050 / 48000)) and np.array_equal(ddelta[:-1], np.diff(dwin))
    for pair in PAIRS:                                  # the package's interleaved table is the oracle's, bit for bit
        t = filter_table(*pair)
        w, d = R.filter_table(*pair)
        assert t.shape == (32769, 2) and np.array_equal(t[:, 0], w) and np.array_equal(t[:, 1], d)


def _tone(f, sr, n, a=0.5):
    return (a * np.sin(2 * np.pi * f * np.arange(n) / sr)).astype(np.float32)


def _mid_rms(y):
    m = y[len(y) // 4: 3 * len(y) // 4].astype(np.float64)
    return float(np.sqrt(np.mean(m * m)))


@pytest.mark.parametrize("sr_orig, sr_new", [(48000, 22050), (44100, 22050), (16000, 22050), (22050, 48000)])
def test_passband_and_stopband(sr_orig, sr_new):
    dc = R.resample(np.full(sr_orig, 0.5, np.float32), sr_orig, sr_new)
    assert float(np.abs(dc[len(dc) // 4: 3 * len(dc) // 4] - 0.5).max()) <= 1e-3
    assert abs(_mid_rms(R.resample(_tone(1000, sr_orig, sr_orig), sr_orig, sr_new)) / (0.5 / np.sqrt(2)) - 1) <= 2e-3
    if sr_new < sr_orig:
        f = 0.55 * sr_new
        assert _mid_rms(R.resample(_tone(f, sr_orig, sr_orig), sr_orig, sr_new)) / (0.5 / np.sqrt(2)) <= 1e-3


@pytest.mark.parametrize("sr_orig, sr_new", [(48000, 22050), (44100, 22050), (22050, 48000), (16000, 22050)])
def test_close_to_torchaudios_kaiser_best_emulation(sr_orig, sr_new):
    TF = pytest.importorskip("torchaudio.functional")
    rng = np.random.default_rng(1)
    x = _tone(440, sr_orig, sr_orig) + (0.05 * rng.standard_normal(sr_orig)).astype(np.float32)
    a = R.resample(x, sr_orig, sr_new)
    b = TF.resample(torch.from_numpy(x).double(), sr_orig, sr_new, lowpass_filter_width=64, rolloff=R.ROLLOFF,
                    resampling_method="sinc_interp_kaiser", beta=R.BETA).numpy()
    k = min(len(a), len(b))
    assert abs(len(a) - len(b)) <= 1
    assert float(np.abs(a[:k] - b[:k]).max()) <= 2e-3
