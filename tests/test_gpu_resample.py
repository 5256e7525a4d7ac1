"""Resampling on the H100 (Resampler, fs2_resample) against the float64 oracle (oracle/resample_oracle.py), bit for bit:
ragged batches with NaN past the lengths at every rate pair in both directions, each utterance against its own B = 1
call, a 60 s input whose running time register crosses about 20 binades, both status bits, `preprocess --resample`
against the oracle's audio through FeatureExtractor, and HiFi-GAN's output taken to 48 kHz."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from conftest import GOLDEN
from fastspeech2_b200 import _lib
from fastspeech2_b200.hparams import load_hp
from fastspeech2_b200.preprocess import gpu_backend, read_wav_np, run
from fastspeech2_b200.resample import Resampler, filter_table, out_length
from oracle import resample_oracle as R

pytestmark = pytest.mark.gpu
FS = 22050
PAIRS = [(48000, FS), (44100, FS), (24000, FS), (16000, FS), (8000, FS)]
PAIRS = PAIRS + [(b, a) for a, b in PAIRS]


def _signal(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    f = 200 + 150 * np.sin(2 * np.pi * 0.3 * t / 22050)
    return (0.3 * np.sin(2 * np.pi * np.cumsum(f) / 22050) + 0.05 * rng.standard_normal(n)).astype(np.float32)


def _batch(xs, fill=float("nan")):
    n = [len(x) for x in xs]
    w = torch.full((len(xs), max(n)), fill)
    for b, x in enumerate(xs):
        w[b, : n[b]] = torch.from_numpy(x)
    return w.cuda(), torch.tensor(n).cuda()


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(np.asarray(a, np.float32).view(np.int32), np.asarray(b, np.float32).view(np.int32))


@pytest.mark.parametrize("sr_orig, sr_new", PAIRS)
def test_ragged_batch_is_the_oracle_bit_for_bit(sr_orig, sr_new):
    r = float(sr_new) / sr_orig
    first = next(n for n in range(1, 100) if int(n * r) >= 1)
    lens = [first, first + 1, 97, 2501, sr_orig // 2, 2 * sr_orig, 10 * sr_orig, 4 * sr_orig + 17, sr_orig + 3]
    xs = [_signal(n, k) for k, n in enumerate(lens)]
    rs = Resampler(sr_orig, sr_new)
    w, n = _batch(xs)
    out, olens = rs(w, n)
    M = out_length(max(lens), sr_orig, sr_new)
    assert out.shape == (len(xs), M) and out.dtype == torch.float32 and olens.dtype == torch.int64
    out, olens = out.cpu().numpy(), olens.cpu().numpy()
    table = R.filter_table(sr_orig, sr_new)
    for b, x in enumerate(xs):
        want = R.resample(x, sr_orig, sr_new, table)
        assert olens[b] == len(want)
        assert _bits_equal(out[b, : olens[b]], want), (b, lens[b])
        assert np.all(out[b, olens[b]:] == 0) and not np.signbit(out[b, olens[b]:]).any()
    for b in (0, 3, 6):                                  # each utterance against its own B = 1 call
        one, ol = rs(*_batch([xs[b]]))
        assert int(ol[0]) == olens[b] and _bits_equal(one[0].cpu().numpy(), out[b, : olens[b]])


def test_a_60_s_input_pins_the_running_time_register():
    x = _signal(60 * 48000, 9)
    out, olens = Resampler(48000, FS)(*_batch([x]))
    want = R.resample(x, 48000, FS)
    assert int(olens[0]) == len(want) == 1323000
    assert _bits_equal(out[0].cpu().numpy(), want)


def _raw(x, lens, sr_orig, sr_new):
    """fs2_resample called directly: -> (y, olens, status) without the module's status check."""
    B, N = x.shape
    M = out_length(N, sr_orig, sr_new)
    n = C.c_size_t()
    _lib.check(_lib.load().fs2_resample_workspace_bytes(B, N, sr_orig, sr_new, M, C.byref(n)), "ws")
    ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
    y = torch.full((B, M), 7.0, device="cuda")
    olens = torch.full((B,), -5, dtype=torch.int64, device="cuda")
    status = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    table = torch.from_numpy(filter_table(sr_orig, sr_new)).cuda()
    _lib.check(_lib.load().fs2_resample(_lib.ptr(x), _lib.ptr(lens), B, N, _lib.ptr(table), sr_orig, sr_new, _lib.ptr(y), _lib.ptr(olens),
                                        M, _lib.ptr(status), _lib.ptr(ws), ws.numel(), _lib.stream_ptr(x.device)), "fs2_resample")
    torch.cuda.synchronize()
    return y.cpu().numpy(), olens.cpu().numpy(), int(status.item())


def test_status_bits_and_what_a_refused_utterance_gets():
    x = _signal(4000, 3)
    w, _ = _batch([x, x, x, x, x])
    lens = torch.tensor([4000, 0, 4001, 2, -3], device="cuda")     # valid; 0; > Nmax; int(2 * 0.459) = 0; negative
    y, olens, status = _raw(w, lens, 48000, FS)
    assert status == _lib.FS2_RS_BAD_LENGTH
    assert olens.tolist() == [out_length(4000, 48000, FS), 0, 0, 0, 0]
    assert _bits_equal(y[0, : olens[0]], R.resample(x, 48000, FS))
    assert np.all(y[1:] == 0) and not np.signbit(y[1:]).any()
    with pytest.raises(ValueError, match=r"every lens\[b\] must lie in \[1, Nmax=4000\]"):
        Resampler(48000, FS)(w, lens)
    bad = x.copy()
    bad[1234] = np.inf
    w2, n2 = _batch([x, bad])
    y, olens, status = _raw(w2, n2, 48000, FS)
    assert status == _lib.FS2_RS_NONFINITE
    with pytest.raises(ValueError, match="finite within lens"):
        Resampler(48000, FS)(w2, n2)
    # NaN (and inf) past lens is never read: the batch helper pads with NaN, here with inf
    w3, n3 = _batch([x[:1000], x], fill=float("inf"))
    y, olens, status = _raw(w3, n3, 22050, 48000)
    assert status == 0 and _bits_equal(y[0, : olens[0]], R.resample(x[:1000], 22050, 48000))


def test_equal_rates_return_the_input():
    w, n = _batch([_signal(100, 0), _signal(50, 1)])
    out, olens = Resampler(FS, FS)(w, n.int())
    assert out is w and olens.dtype == torch.int64 and torch.equal(olens, n)


def _golden_wavs():
    return [read_wav_np(os.path.join(GOLDEN, f), FS) for f in ("sample_58k.wav", "sample_74k_waveglow.wav")]


def test_preprocess_resample_matches_the_oracle_through_the_feature_extractor(tmp_path):
    root = tmp_path / "wavs48"
    root.mkdir()
    up = [R.resample(w, FS, 48000) for w in _golden_wavs()]
    i16 = [np.round(np.clip(u, -1, 1) * 32767).astype(np.int16) for u in up]
    wavfile.write(str(root / "a.wav"), 48000, i16[0])
    wavfile.write(str(root / "b.wav"), 48000, np.stack([i16[1], (i16[1] // 2).astype(np.int16)], 1))   # stereo
    hp = load_hp()
    res = run(str(root), hp, str(tmp_path / "out"), budget=1 << 22, log=lambda *a: None, resample=True)
    assert res["ids"] == ["a", "b"]
    extract = gpu_backend(hp)
    for uid in ("a", "b"):
        sr, w = read_wav_np(str(root / f"{uid}.wav"), FS, resample=True)
        assert sr == 48000
        mel, e, p = extract([R.resample(w, 48000, FS)])[0]
        for d, want in (("mels", mel), ("energy", e)):
            assert _bits_equal(np.load(tmp_path / "out" / d / f"{uid}.npy"), want), (uid, d)
        assert np.array_equal(np.load(tmp_path / "out" / "pitch" / f"{uid}.npy"), p)


def test_a_native_rate_tree_is_byte_identical_with_and_without_resample(tmp_path):
    root = tmp_path / "wavs"
    root.mkdir()
    for uid, w in zip(("a", "b"), _golden_wavs()):
        wavfile.write(str(root / f"{uid}.wav"), FS, np.round(w * 32767).astype(np.int16))
    hp = load_hp()
    for flag in (False, True):
        run(str(root), hp, str(tmp_path / str(flag)), stats=True, log=lambda *a: None, resample=flag)
    for d in ("mels", "energy", "pitch"):
        for uid in ("a", "b"):
            a, b = (open(tmp_path / str(f) / d / f"{uid}.npy", "rb").read() for f in (False, True))
            assert a == b, (d, uid)
    for k in ("e_mean", "e_std", "f0_mean", "f0_std"):
        assert open(tmp_path / "False" / f"{k}.npy", "rb").read() == open(tmp_path / "True" / f"{k}.npy", "rb").read()


def test_hifigan_audio_to_48_khz_is_the_oracle():
    from fastspeech2_b200.hifigan import HiFiGANVocoder
    torch.manual_seed(0)
    v = HiFiGANVocoder("v3").cuda()
    olens = torch.tensor([40, 17, 63], device="cuda")
    mels = (torch.randn(3, 63, 80, generator=torch.Generator().manual_seed(2)) * 2 - 6).cuda()
    with torch.no_grad():
        audio, alens = v(mels, olens)
        out, ol = Resampler(FS, 48000)(audio, alens)
    audio, alens, out, ol = audio.cpu().numpy(), alens.cpu().numpy(), out.cpu().numpy(), ol.cpu().numpy()
    for b in range(3):
        want = R.resample(audio[b, : alens[b]], FS, 48000)
        assert ol[b] == len(want) and _bits_equal(out[b, : ol[b]], want)
        assert np.all(out[b, ol[b]:] == 0)
