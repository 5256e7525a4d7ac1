"""Training features without a GPU: the float64 DIO oracle tracks pitch, its formulas (bands, fft_size, f0_length), its
mel and energy against an independent float64 STFT, the statistics restatement, the preprocessing command with the oracle
as its backend, the library's workspace formula, argument validation and the C entry points."""
import glob
import math
import os
import re

import numpy as np
import pytest
import torch

from conftest import REPO
from fastspeech2_b200 import _lib
from fastspeech2_b200.features import FeatureExtractor
from fastspeech2_b200.hparams import AttrDict, load_hp
from fastspeech2_b200.preprocess import read_wav_np, remove_outlier, run, statistics
from fastspeech2_b200.vocoder import mel_filterbank
from oracle import dio_oracle as D

FS, HOP = 22050, 256
FP = D.frame_period_ms(HOP, FS)


def _harmonic(f0_of_t, n, seed, noise=1e-3):
    rng = np.random.default_rng(seed)
    ph = 2 * np.pi * np.cumsum(f0_of_t(np.arange(n) / FS)) / FS
    return sum((0.3 / k) * np.sin(k * ph + k) for k in range(1, 6)) + noise * rng.standard_normal(n)


def _interior(f0, margin=6):
    v = np.flatnonzero(f0 > 0)
    return v[(v >= v.min() + margin) & (v <= v.max() - margin)]


def test_dio_tracks_a_steady_150_hz_tone():
    f0 = D.dio(_harmonic(lambda t: np.full_like(t, 150.0), 2 * FS, 0), FS, frame_period=FP)
    idx = _interior(f0)
    assert len(idx) > 0.8 * len(f0)
    assert float(np.max(np.abs(f0[idx] / 150.0 - 1))) <= 0.01


def test_dio_tracks_a_100_to_300_hz_glide():
    n = 2 * FS
    f_true = lambda t: 100.0 * 3.0 ** (t / (n / FS))                   # noqa: E731
    f0 = D.dio(_harmonic(f_true, n, 1), FS, frame_period=FP)
    idx = _interior(f0)
    assert len(idx) > 0.8 * len(f0)
    assert float(np.max(np.abs(f0[idx] / f_true(idx * FP / 1000.0) - 1))) <= 0.02


@pytest.mark.parametrize("amp", [1e-3, 0.3])
def test_dio_calls_noise_and_dithered_silence_unvoiced(amp):
    x = amp * np.random.default_rng(2).standard_normal(2 * FS)
    f0 = D.dio(x, FS, frame_period=FP)
    assert np.mean(f0 == 0) >= 0.95


def test_dio_short_contours_are_all_zero():
    for n in (513, 600, 700):                      # f0_length = 3 <= vrm = 3
        assert D.f0_length(n, FS, FP) <= 3
        f0 = D.dio(_harmonic(lambda t: np.full_like(t, 150.0), n, 3), FS, frame_period=FP)
        assert len(f0) == D.f0_length(n, FS, FP) and np.all(f0 == 0)


def test_formulas():
    b = D.band_edges()
    assert len(b) == 7 and np.allclose(b, 71.0 * 2.0 ** (np.arange(1, 8) / 2.0), rtol=0, atol=0)
    assert D.matlab_round(FS / b[0] / 2.0) == 110 and D.matlab_round(FS / 50.0) == 441
    assert len(D.lowcut_taps(FS)) == 883 and abs(float(D.lowcut_taps(FS).sum())) < 1e-12
    # fft_size: the smallest power of two strictly greater than y_length + 440
    for n in (1000, 32767 - 441, 32767 - 440, 108288):
        F = D.fft_size(n, FS, b[0])
        assert F > n + 1 + 440 >= F // 2
    assert D.fft_size(32326, FS, b[0]) == 32768 and D.fft_size(32327, FS, b[0]) == 65536   # 32767 and 32768 samples
    # WORLD computes the size as 2^(int(log(m) / kLog2) + 1); that is exact at every power of two
    assert all(int(math.log(2.0 ** k) / D.K_LOG2) == k for k in range(1, 31))
    # f0_length = int(1000 N / fs / frame_period) + 1 is one frame short of T = N // hop + 1 at some multiples of hop
    assert D.f0_length(3328, FS, FP) == 13 and 3328 // HOP + 1 == 14
    short = [n for n in range(HOP, 2_000_000, HOP) if D.f0_length(n, FS, FP) < n // HOP + 1]
    assert len(short) == 343 and short[0] == 3328
    assert all(D.f0_length(n, FS, FP) <= n // HOP + 1 for n in range(1, 100000))


def _np_mel_energy(x, n_fft=1024, hop=256, n_mels=80):
    """float64 numpy: reflect pad, periodic Hann frames, rfft, mel filterbank, log(clamp)."""
    x = np.pad(np.asarray(x, np.float64), n_fft // 2, mode="reflect")
    T = (len(x) - n_fft) // hop + 1
    win = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(n_fft) / n_fft)
    fr = np.stack([x[t * hop: t * hop + n_fft] * win for t in range(T)])
    mag = np.abs(np.fft.rfft(fr, axis=1)).T
    basis = mel_filterbank(FS, n_fft, n_mels, 0.0, 8000.0).astype(np.float64)
    return np.log(np.maximum(basis @ mag, 1e-5)), np.sqrt((mag ** 2).sum(axis=0))


def test_oracle_mel_and_energy_are_the_reference_transform():
    from oracle.stft_oracle import STFT
    x = (0.5 * _harmonic(lambda t: 130 + 40 * t, 20000, 4)).astype(np.float32)
    mel, e = D.mel_energy(x)
    assert mel.shape == (80, 20000 // HOP + 1) and e.shape == (20000 // HOP + 1,)
    mag, _ = STFT(1024, 256, 1024).transform(torch.from_numpy(x)[None])
    basis = torch.from_numpy(mel_filterbank(FS, 1024, 80, 0.0, 8000.0))
    assert np.array_equal(mel, torch.log(torch.clamp(basis @ mag[0], min=1e-5)).numpy())
    assert np.array_equal(e, torch.norm(mag[0], dim=0).numpy())
    m64, e64 = _np_mel_energy(x)
    assert float(np.abs(e - e64).max()) <= 1e-5 * float(e64.max())
    big = np.exp(m64) > 1e-3 * np.exp(m64).max(axis=0, keepdims=True)
    assert float(np.abs(mel - m64)[big].max()) <= 1e-3


def test_remove_outlier_restatement():
    x = np.array([1.0, 2.0, 2.0, 3.0, 0.0, 2.5, 100.0, 2.0, -50.0], dtype=np.float32)
    # p25 = 1, p75 = 2.5: fences -1.25 and 4.75; 100 and -50 are outliers, set to 0, then to max(x) = 3; 0 stays 0
    got = remove_outlier(x.copy())
    assert np.array_equal(got, np.array([1, 2, 2, 3, 0, 2.5, 3, 2, 3], dtype=np.float32)) and got.dtype == np.float32
    y = np.array([5.0, 5.0, 5.0, 5.0])                 # zero IQR: every value sits on a fence, then max = 0
    assert np.array_equal(remove_outlier(y), np.zeros(4))


def test_statistics_restatement():
    lines = []
    e = {"a": np.array([1.0, 2.0, 3.0, 0.0], np.float32), "b": np.array([2.0, 4.0, 2.0, 3.0], np.float32)}
    p = {"a": np.array([0.0, 100.0, 110.0, 120.0, 0.0]), "b": np.zeros(4)}
    st = statistics(e, p, log=lambda *a: lines.append(" ".join(str(v) for v in a)))
    nz_e = np.array([1, 2, 3, 2, 4, 2, 3], np.float32)
    assert st["e_mean"] == np.float32(np.mean(nz_e)) and st["e_std"] == np.float32(np.std(nz_e))
    assert abs(float(st["f0_mean"]) - 110.0) < 1e-5 and abs(float(st["f0_std"]) - np.std([100.0, 110, 120])) < 1e-5
    assert st["bad_pitch"] == ["b"] and st["e_mean"].dtype == np.float32
    assert "Max Energy : 4.0" in lines and "Min Pitch : 0.0" in lines and lines[-1] == "b"


def _write_wavs(d):
    from scipy.io import wavfile
    rng = np.random.default_rng(5)
    x = (0.5 * _harmonic(lambda t: np.full_like(t, 140.0), 9000, 6)).astype(np.float32)
    (d / "sub").mkdir(parents=True)
    wavfile.write(str(d / "a.wav"), FS, np.round(x * 32767).astype(np.int16))
    wavfile.write(str(d / "sub" / "b.x.wav"), FS, np.stack([x[:7000], rng.standard_normal(7000).astype(np.float32)], 1))
    wavfile.write(str(d / "c.wav"), FS, np.round(x[:5000] * 127 + 128).astype(np.uint8))
    wavfile.write(str(d / "d.wav"), FS, np.round(x[:6000] * 2 ** 31).astype(np.int32))
    return x


def test_read_wav_np_rules(tmp_path):
    x = _write_wavs(tmp_path)
    a = read_wav_np(str(tmp_path / "a.wav"), FS)
    assert a.dtype == np.float32 and np.abs(a - x).max() <= 1 / 32768
    b = read_wav_np(str(tmp_path / "sub" / "b.x.wav"), FS)
    assert np.array_equal(b, x[:7000])                                # the first channel
    c = read_wav_np(str(tmp_path / "c.wav"), FS)
    assert np.abs(c - x[:5000]).max() <= 1 / 128
    d = read_wav_np(str(tmp_path / "d.wav"), FS)
    assert np.abs(d - x[:6000]).max() <= 1e-6
    with pytest.raises(ValueError, match="sample rate"):
        read_wav_np(str(tmp_path / "a.wav"), 16000)


def test_preprocess_command_with_the_oracle_backend(tmp_path):
    _write_wavs(tmp_path / "wavs")
    hp = AttrDict({"audio": dict(load_hp().audio), "data": {"data_dir": str(tmp_path / "out")}})
    lines = []
    res = run(str(tmp_path / "wavs"), hp, stats=True, budget=15000, extract=lambda ws: [D.features(w) for w in ws],
              log=lambda *a: lines.append(" ".join(str(v) for v in a)))
    assert sorted(res["ids"]) == ["a", "b", "c", "d"]
    for k, n in (("a", 9000), ("b", 7000), ("c", 5000), ("d", 6000)):
        T = n // HOP + 1
        m = np.load(tmp_path / "out" / "mels" / f"{k}.npy")
        e = np.load(tmp_path / "out" / "energy" / f"{k}.npy")
        p = np.load(tmp_path / "out" / "pitch" / f"{k}.npy")
        assert m.dtype == np.float32 and m.shape == (80, T)
        assert e.dtype == np.float32 and e.shape == (T,)
        assert p.dtype == np.float64 and p.shape == (min(D.f0_length(n, FS, FP), T),)
        assert np.any(p > 0)
    for k in ("e_mean", "e_std", "f0_mean", "f0_std"):
        v = np.load(tmp_path / "out" / f"{k}.npy")
        assert v.dtype == np.float32 and v.shape == () and v > 0
    assert any(s.startswith("Pitch mean : ") for s in lines)
    hp.audio["sample_rate"] = 16000
    with pytest.raises(ValueError, match="sample rate"):
        run(str(tmp_path / "wavs"), hp, str(tmp_path / "out2"), extract=lambda ws: [], log=lambda *a: None)


def _round(n):
    return (n + 255) // 256 * 256


def _workspace_formula(B, N, sr=22050, n_fft=1024, hop=256, n_mels=80, f0_floor=71.0, cio=2.0, f0_ceil=800.0):
    cutoff = n_fft // 2 + 1
    cpad, mpad = (2 * cutoff + 63) // 64 * 64, (cutoff + 63) // 64 * 64
    T, Tp = N // hop + 1, N // hop + 2
    P = 2 * D.matlab_round(sr / (f0_floor * 2 ** (1 / cio)) / 2)
    nb = len(D.band_edges(f0_floor, f0_ceil, cio))
    mel = sum(_round(v) for v in (B * T * n_fft * 4, B * T * cpad * 4, B * T * mpad * 4, B * T * n_mels * 4, B * 8))
    dio = sum(_round(v) for v in (B * 24, B * (N + 1 + 2 * P) * 8, B * (N + 2) * 8, 4 * B * (N // 2 + 2) * 8, 4 * B * 4,
                                  nb * B * Tp * 8, B * Tp * 8, B * Tp * 8, B * Tp * 8, B * Tp * 8))
    return max(mel, dio) + 256


@pytest.mark.parametrize("B,N", [(1, 600), (3, 50000), (64, 220500), (7, 4096 * 256)])
def test_workspace_formula(B, N):
    fx = FeatureExtractor()
    n = fx.workspace_bytes(B, N)
    assert n == _workspace_formula(B, N)
    assert n <= 48 * B * N + 16384 * B + 4096
    f2 = FeatureExtractor(16000, 512, 128, 512, 64, 55.0, 7600.0, math_mode="fp32")
    assert f2.workspace_bytes(B, N) == _workspace_formula(B, N, 16000, 512, 128, 64)


def test_hp_plumbing():
    f = FeatureExtractor.from_hp(load_hp())
    assert (f.sample_rate, f.n_fft, f.hop_length, f.win_length, f.n_mels, f.fmin, f.fmax) == (22050, 1024, 256, 1024, 80, 0.0, 8000.0)
    assert f.math_mode == "3xf16" and f.frame_period == 256 / 22050 * 1000
    assert (f.f0_floor, f.f0_ceil, f.channels_in_octave, f.allowed_range) == (71.0, 800.0, 2.0, 0.1)
    assert torch.equal(f.mel_basis, torch.from_numpy(mel_filterbank(22050, 1024, 80, 0.0, 8000.0)))
    with pytest.raises(ValueError, match="math_mode"):
        FeatureExtractor(math_mode="bf16")


@pytest.mark.parametrize("wavs,lens,match", [
    (torch.zeros(2, 1000, 1), torch.tensor([1000, 900]), r"\[B, Nmax\]"),
    (torch.zeros(0, 1000), torch.tensor([], dtype=torch.long), r"\[B, Nmax\]"),
    (torch.zeros(2, 1000, dtype=torch.float64), torch.tensor([1000, 900]), "float32"),
    (torch.zeros(2, 1000), torch.tensor([1000]), "lens"),
    (torch.zeros(2, 1000), torch.tensor([1000.0, 900.0]), "integer"),
    (torch.zeros(2, 1000), torch.tensor([True, False]), "integer"),
    (torch.zeros(2, 500), torch.tensor([500, 500]), "too short"),
    (torch.zeros(2, 1000), torch.tensor([1000, 900]), "CUDA")])
def test_bad_inputs_raise(wavs, lens, match):
    fx = FeatureExtractor()
    for call in (fx.mel_energy, fx.pitch, fx):
        with pytest.raises(ValueError, match=match):
            call(wavs, lens)


def test_library_exports_feature_entry_points():
    lib = _lib.load()
    header = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    for name in ("fs2_features_create", "fs2_features_load", "fs2_features_workspace_bytes", "fs2_mel_energy", "fs2_dio"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES, name
        assert f"int {name}(" in header, name
    assert hasattr(lib, "fs2_features_destroy") and "void fs2_features_destroy(" in header


def test_create_rejects_bad_configs():
    import ctypes as C
    lib = _lib.load()
    good = dict(sample_rate=22050, n_fft=1024, hop=256, win_length=1024, n_mels=80, math_mode=2, f0_floor=71.0, f0_ceil=800.0,
                channels_in_octave=2.0, allowed_range=0.1)
    for bad in (dict(n_fft=1000), dict(hop=600), dict(n_mels=70), dict(math_mode=9), dict(f0_ceil=50.0), dict(f0_floor=0.0),
                dict(channels_in_octave=8.0), dict(sample_rate=500)):
        cfg = _lib.FeaturesConfig(**{**good, **bad})
        h = C.c_void_p()
        assert lib.fs2_features_create(C.byref(h), C.byref(cfg)) != 0, bad
    h = C.c_void_p()
    assert lib.fs2_features_create(C.byref(h), C.byref(_lib.FeaturesConfig(**good))) == 0
    lib.fs2_features_destroy(h)


def test_feature_kernels_do_not_spill():
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "features.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = open(reports[0]).read()
    for kernel in ("feat_frames_kernel", "feat_magnitude_kernel", "feat_log_kernel", "dio_prepare_kernel", "dio_lowcut_kernel",
                   "dio_band_kernel", "dio_events_kernel", "dio_frames_kernel", "dio_fix_kernel"):
        props = re.findall(r"Function properties for \S*%s\S*\n(.*)" % kernel, text)
        assert props, kernel
        for line in props:
            assert "0 bytes spill stores, 0 bytes spill loads" in line, (kernel, line)
