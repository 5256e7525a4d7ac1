"""Resampling without a device: Resampler's argument checks, the C entries' size checks and workspace formula, the
kernels' register report, read_wav_np's resample branch, and `preprocess --resample` batching runs of one rate with
the oracle as its resampling hook."""
import ctypes as C
import glob
import os
import re

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from conftest import REPO
from fastspeech2_b200 import _lib
from fastspeech2_b200.hparams import AttrDict, load_hp
from fastspeech2_b200.preprocess import main, read_wav_np, run
from fastspeech2_b200.resample import Resampler, out_length, workspace_bytes
from oracle import resample_oracle as R

FS, HOP = 22050, 256


@pytest.mark.parametrize("change, match", [
    (lambda a: {"wavs": a["wavs"][0]}, r"wavs must be a non-empty \[B, Nmax\]"),
    (lambda a: {"wavs": a["wavs"][:, :0]}, "wavs must be a non-empty"),
    (lambda a: {"wavs": a["wavs"].double()}, "wavs must be float32"),
    (lambda a: {"lens": a["lens"][:1]}, r"lens must be a \[B=2\] tensor"),
    (lambda a: {"lens": a["lens"].float()}, "lens must be an integer tensor"),
    (lambda a: {"lens": a["lens"].bool()}, "lens must be an integer tensor"),
    (lambda a: {}, "wavs and lens must be CUDA tensors"),
])
def test_forward_argument_checks(change, match):
    a = {"wavs": torch.zeros(2, 100), "lens": torch.full((2,), 100)}
    a.update(change(a))
    with pytest.raises(ValueError, match=match):
        Resampler(48000, 22050)(a["wavs"], a["lens"])


@pytest.mark.parametrize("orig, new, match", [
    (0, 22050, "orig_sr must be an integer sample rate"),
    (48000.0, 22050, "orig_sr must be an integer"),
    (True, 22050, "orig_sr must be an integer"),
    (22050, 1 << 25, "new_sr must be an integer sample rate"),
    (600000, 1000, "more than 512"),
])
def test_constructor_checks(orig, new, match):
    with pytest.raises(ValueError, match=match):
        Resampler(orig, new)


def test_equal_rates_still_check_their_arguments():
    with pytest.raises(ValueError, match="CUDA tensors"):
        Resampler(22050, 22050)(torch.zeros(1, 5), torch.tensor([5]))


def _ws(*args):
    n = C.c_size_t()
    return _lib.load().fs2_resample_workspace_bytes(*args, C.byref(n)), n.value


def test_workspace_formula():
    a256 = lambda v: (v + 255) // 256 * 256     # noqa: E731
    for B, N, so, sn in ((1, 1000, 48000, 22050), (64, 480000, 48000, 22050), (9, 220500, 22050, 48000), (3, 7, 8000, 22050)):
        M = out_length(N, so, sn)
        assert M == int(np.ceil(N * (sn / so)))
        assert _ws(B, N, so, sn, M) == (0, a256(8 * B * M) + 256)
        assert workspace_bytes(B, N, so, sn) == a256(8 * B * M) + 256
        assert _ws(B, N, so, sn, M + 10)[1] == a256(8 * B * (M + 10)) + 256


@pytest.mark.parametrize("args, match", [
    ((0, 5, 48000, 22050, 3), r"B \(0\)"),
    ((1, 0, 48000, 22050, 3), r"Nmax \(0\)"),
    ((1, 5, 0, 22050, 3), "sample rates"),
    ((1, 5, 48000, (1 << 24) + 1, 3), "sample rates"),
    ((1, 5, 22050, 22050, 5), "equal sample rates"),
    ((1, 5, 600000, 1000, 1), "more than 512"),
    ((1, 5, 48000, 22050, 2), r"Mmax \(2\) must lie in \[ceil\(Nmax \* ratio\) = 3"),
    ((1, 1 << 26, 22050, 48000, (1 << 26) - 1), "Mmax"),
])
def test_c_size_checks(args, match):
    rc, _ = _ws(*args)
    assert rc == -1
    assert re.search(match, _lib.load().fs2_last_error().decode())


def test_c_entry_refuses_null_arguments_without_a_gpu():
    lib = _lib.load()
    assert lib.fs2_resample(None, None, 1, 5, None, 48000, 22050, None, None, 3, None, None, 0, None) == -1
    assert "null argument" in lib.fs2_last_error().decode()
    assert lib.fs2_resample_workspace_bytes(1, 5, 48000, 22050, 3, None) == -1


def test_resample_kernels_do_not_spill():
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "resample.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = open(reports[0]).read()
    for kernel in ("rs_clock_kernel", "rs_taps_kernel"):
        props = re.findall(r"Function properties for \S*%s\S*\n(.*)" % kernel, text)
        assert props, kernel
        for line in props:
            assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in line, (kernel, line)


# ---- reading and preprocessing ----------------------------------------------------------------------------------------

def _signal(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    return (0.4 * np.sin(2 * np.pi * 0.013 * t) + 0.05 * rng.standard_normal(n)).astype(np.float32)


def test_read_wav_np_resample_branch(tmp_path):
    x, z = _signal(4000, 1), _signal(4000, 2)
    s16 = np.round(np.stack([x, z], 1) * 32767).astype(np.int16)
    wavfile.write(str(tmp_path / "st.wav"), 48000, s16)
    sr, w = read_wav_np(str(tmp_path / "st.wav"), FS, resample=True)
    assert sr == 48000 and w.dtype == np.float32 and w.shape == (4000,)
    y = (s16 / 32768.0).astype(np.float32)
    assert np.array_equal(w, np.mean(y.T, axis=0))                  # the channel mean, not the first channel
    wavfile.write(str(tmp_path / "u8.wav"), 16000, np.round(x * 127 + 128).astype(np.uint8))
    sr, w = read_wav_np(str(tmp_path / "u8.wav"), FS, resample=True)
    assert sr == 16000 and np.array_equal(w, ((np.round(x * 127 + 128) - 128) / 128.0).astype(np.float32))
    wavfile.write(str(tmp_path / "i32.wav"), 44100, np.round(x.astype(np.float64) * 2 ** 30).astype(np.int32))
    sr, w = read_wav_np(str(tmp_path / "i32.wav"), FS, resample=True)
    assert sr == 44100 and np.abs(w - x / 2).max() <= 1e-6
    wavfile.write(str(tmp_path / "nat.wav"), FS, s16)                # at the configured rate: the first channel, as before
    sr, w = read_wav_np(str(tmp_path / "nat.wav"), FS, resample=True)
    assert sr == FS and np.array_equal(w, read_wav_np(str(tmp_path / "nat.wav"), FS)) and np.array_equal(w, y[:, 0])
    bad = x.copy()
    bad[7] = np.nan
    wavfile.write(str(tmp_path / "nan.wav"), 24000, bad)
    with pytest.raises(ValueError, match="not finite"):
        read_wav_np(str(tmp_path / "nan.wav"), FS, resample=True)
    with pytest.raises(ValueError, match="sample rate 48000 Hz.*--resample"):
        read_wav_np(str(tmp_path / "st.wav"), FS)


def _tree(root):
    """Sorted names a..f: rates 48k, 48k, 22.05k, 48k, 16k, 16k, so four runs of one rate."""
    spec = [("a", 48000, 9000), ("b", 48000, 12000), ("c", FS, 5000), ("d", 48000, 3000), ("e", 16000, 4000), ("f", 16000, 6000)]
    os.makedirs(root)
    for k, (uid, sr, n) in enumerate(spec):
        wavfile.write(os.path.join(root, uid + ".wav"), sr, np.round(_signal(n, k) * 32767).astype(np.int16))
    return spec


def _features(w):
    T = len(w) // HOP + 1
    return np.full((80, T), float(len(w)), np.float32), np.arange(T, dtype=np.float32), np.zeros(T - 1)


def test_run_resamples_runs_of_one_rate_with_the_hook(tmp_path):
    spec = _tree(str(tmp_path / "wavs"))
    hp = AttrDict({"audio": dict(load_hp().audio), "data": {"data_dir": str(tmp_path / "out")}})
    calls, extracted = [], []

    def hook(wavs, orig, new):
        calls.append((orig, new, len(wavs)))
        return R.backend(wavs, orig, new)

    def extract(ws):
        extracted.append([len(w) for w in ws])
        return [_features(w) for w in ws]
    res = run(str(tmp_path / "wavs"), hp, budget=40000, extract=extract, log=lambda *a: None, resample=hook)
    assert res["ids"] == ["a", "b", "c", "d", "e", "f"]
    assert calls == [(48000, FS, 2), (48000, FS, 1), (16000, FS, 2)]
    want = {uid: out_length(n, sr, FS) for uid, sr, n in spec}
    assert want["c"] == 5000 and want["a"] == int(np.ceil(9000 * FS / 48000))
    assert extracted == [[want["a"], want["b"]], [want["c"]], [want["d"]], [want["e"], want["f"]]]
    for uid, _, _ in spec:
        m = np.load(tmp_path / "out" / "mels" / f"{uid}.npy")
        assert m.shape == (80, want[uid] // HOP + 1) and m[0, 0] == want[uid]
    # the extractor sees the oracle's audio, and a run that splits at the budget gives the same files
    wav_a = read_wav_np(str(tmp_path / "wavs" / "a.wav"), FS, resample=True)[1]
    seen = []
    run(str(tmp_path / "wavs"), hp, str(tmp_path / "out2"), budget=1, extract=lambda ws: seen.extend(ws) or [_features(w) for w in ws],
        log=lambda *a: None, resample=R.backend)
    assert np.array_equal(seen[0], R.resample(wav_a, 48000, FS))
    for uid, _, _ in spec:
        assert np.array_equal(np.load(tmp_path / "out" / "mels" / f"{uid}.npy"), np.load(tmp_path / "out2" / "mels" / f"{uid}.npy"))


def test_budget_bounds_the_resampled_batch(tmp_path):
    root = str(tmp_path / "wavs")
    os.makedirs(root)
    for uid in ("a", "b"):
        wavfile.write(os.path.join(root, uid + ".wav"), 8000, np.round(_signal(1000, 0) * 32767).astype(np.int16))
    hp = AttrDict({"audio": dict(load_hp().audio), "data": {"data_dir": str(tmp_path / "out")}})
    sizes = []
    hook = lambda ws, o, n: sizes.append(len(ws)) or R.backend(ws, o, n)     # noqa: E731
    up = out_length(1000, 8000, FS)                                         # 2757 samples after resampling
    run(root, hp, budget=2 * up - 1, extract=lambda ws: [_features(w) for w in ws], log=lambda *a: None, resample=hook)
    assert sizes == [1, 1]                                                  # 2 * 1000 fits, 2 * 2757 does not
    sizes.clear()
    run(root, hp, budget=2 * up, extract=lambda ws: [_features(w) for w in ws], log=lambda *a: None, resample=hook)
    assert sizes == [2]


def test_default_path_still_refuses_other_rates(tmp_path, monkeypatch):
    _tree(str(tmp_path / "wavs"))
    hp = AttrDict({"audio": dict(load_hp().audio), "data": {"data_dir": str(tmp_path / "out")}})
    with pytest.raises(ValueError, match="sample rate"):
        run(str(tmp_path / "wavs"), hp, extract=lambda ws: [_features(w) for w in ws], log=lambda *a: None)
    got = {}
    monkeypatch.setattr("fastspeech2_b200.preprocess.run", lambda *a, **k: got.update(args=a, kw=k))
    cfg = os.path.join(REPO, "fastspeech2_b200", "configs", "default.yaml")
    main(["-d", "x", "-c", cfg])
    assert got["kw"]["resample"] is False
    main(["-d", "x", "-c", cfg, "--resample"])
    assert got["kw"]["resample"] is True
