"""Batched Griffin-Lim vocoder without a GPU: the package's mel filterbank against torchaudio's independent one, the CPU
oracle against the reference-loop oracle and against torchaudio's griffinlim, hp plumbing, argument validation, and the
C entry points."""
import glob
import os
import re

import numpy as np
import pytest
import torch

from conftest import REPO
from fastspeech2_b200 import _lib
from fastspeech2_b200.hparams import AttrDict, load_hp
from fastspeech2_b200.vocoder import GriffinLimVocoder, mel_filterbank, mel_inverse
from oracle import gl_oracle as G
from oracle import stft_oracle as O


@pytest.mark.parametrize("sr,n_fft,n_mels,fmin,fmax", [(22050, 1024, 80, 0.0, 8000.0), (16000, 512, 64, 55.0, 7600.0)])
def test_mel_filterbank_matches_torchaudio(sr, n_fft, n_mels, fmin, fmax):
    import torchaudio.functional as TAF
    ours = mel_filterbank(sr, n_fft, n_mels, fmin, fmax)
    ta = TAF.melscale_fbanks(n_fft // 2 + 1, fmin, fmax, n_mels, sr, norm="slaney", mel_scale="slaney").T.numpy()
    assert ours.shape == (n_mels, n_fft // 2 + 1) and ours.dtype == np.float32
    assert float(np.abs(ours - ta).max()) <= 1e-6
    P = mel_inverse(ours)
    assert P.shape == (n_fft // 2 + 1, n_mels) and P.dtype == np.float32
    assert np.allclose(ours.astype(np.float64) @ P.astype(np.float64), np.eye(n_mels), atol=1e-4)


def _harmonic(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n) / 22050.0
    return (0.4 * torch.sin(2 * np.pi * 220 * t) + 0.2 * torch.sin(2 * np.pi * 1330 * t + 0.3))[None] + 0.01 * torch.randn(1, n, generator=g)


def test_oracle_without_momentum_is_the_reference_loop():
    st = O.STFT(1024, 256, 1024)
    mag, _ = st.transform(_harmonic(60 * 256))
    angles = (torch.rand(mag.shape, generator=torch.Generator().manual_seed(3)) * 2 - 1) * np.pi
    for n_iters in (0, 3):
        assert torch.equal(G.griffin_lim(mag, st, n_iters, angles), O.griffin_lim(mag, st, n_iters, angles))


@pytest.mark.parametrize("momentum", [0.0, 0.99])
@pytest.mark.parametrize("n_iters", [1, 4])
def test_oracle_agrees_with_torchaudio_griffinlim(momentum, n_iters):
    import torchaudio.functional as TAF
    n = 119 * 256
    st = O.STFT(1024, 256, 1024)
    mag, _ = st.transform(_harmonic(n))
    ours = G.griffin_lim(mag, st, n_iters, torch.zeros_like(mag), momentum)
    win = torch.hann_window(1024, periodic=True, dtype=torch.float64)
    ta = TAF.griffinlim(mag.double(), win, 1024, 256, 1024, 1.0, n_iters, momentum, n, False).float()
    assert ours.shape == ta.shape
    assert float((ours - ta).abs().max()) <= 5e-4 * float(ta.abs().max())


def test_hp_plumbing():
    v = GriffinLimVocoder.from_hp(load_hp())
    assert (v.sample_rate, v.n_fft, v.hop_length, v.win_length, v.n_mels, v.fmin, v.fmax) == (22050, 1024, 256, 1024, 80, 0.0, 8000.0)
    assert v.cutoff == 513 and tuple(v.mel_inverse.shape) == (513, 80) and v.math_mode == "3xf16"
    assert torch.equal(v.mel_basis, torch.from_numpy(mel_filterbank(22050, 1024, 80, 0.0, 8000.0)))
    # the reference's config names the mel count num_mels (configs/default.yaml carries both)
    a = AttrDict({"audio": {"sample_rate": 16000, "n_fft": 512, "hop_length": 128, "win_length": 400, "num_mels": 64,
                            "fmin": 55.0, "fmax": 7600.0}})
    v = GriffinLimVocoder.from_hp(a, math_mode="fp32")
    assert (v.sample_rate, v.n_fft, v.hop_length, v.win_length, v.n_mels, v.math_mode) == (16000, 512, 128, 400, 64, "fp32")
    assert tuple(v.stft.forward_basis.shape) == (514, 1, 512) and v.cutoff == 257
    with pytest.raises(ValueError, match="math_mode"):
        GriffinLimVocoder(math_mode="bf16")


@pytest.fixture(scope="module")
def voc():
    return GriffinLimVocoder()


@pytest.mark.parametrize("kw,match", [
    (dict(n_iters=-1), "n_iters"), (dict(n_iters=2.0), "n_iters"), (dict(momentum=1.0), "momentum"),
    (dict(momentum=-0.1), "momentum"), (dict(seed=1.5), "seed"), (dict(seed=torch.zeros(3, dtype=torch.long)), "seed")])
def test_bad_arguments_raise(voc, kw, match):
    with pytest.raises(ValueError, match=match):
        voc(torch.zeros(2, 10, 80), torch.tensor([10, 9]), **kw)


@pytest.mark.parametrize("shape,olens,match", [
    ((2, 10), [10, 9], "mels"), ((2, 10, 40), [10, 9], "mels"), ((2, 10, 80), [10], "olens"),
    ((2, 10, 80), [10.0, 9.0], "integer"), ((2, 2, 80), [2, 2], "too short"), ((2, 10, 80), [10, 9], "CUDA")])
def test_bad_inputs_raise(voc, shape, olens, match):
    with pytest.raises(ValueError, match=match):
        voc(torch.zeros(shape), torch.tensor(olens))
    with pytest.raises(ValueError, match=match):
        voc.mel_to_magnitude(torch.zeros(shape), torch.tensor(olens))


def test_library_exports_vocoder_entry_points():
    lib = _lib.load()
    header = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    for name in ("fs2_vocoder_create", "fs2_vocoder_load", "fs2_vocoder_workspace_bytes", "fs2_mel_magnitude", "fs2_griffin_lim"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES, name
        assert f"int {name}(" in header, name
    assert hasattr(lib, "fs2_vocoder_destroy") and "void fs2_vocoder_destroy(" in header


def test_vocoder_kernels_do_not_spill():
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "griffin_lim.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = open(reports[0]).read()
    for kernel in ("mel_expand_kernel", "gl_project_kernel", "ola_frame_kernel", "ola_audio_kernel", "mag_transpose_kernel"):
        props = re.findall(r"Function properties for \S*%s\S*\n(.*)" % kernel, text)
        assert props, kernel
        for line in props:
            assert "0 bytes spill stores, 0 bytes spill loads" in line, (kernel, line)
