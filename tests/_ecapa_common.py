"""Shared pieces of the ECAPA-TDNN GPU tests: 16 kHz test audio, seeded and calibrated oracle models, float64 references."""
import functools
import os

import numpy as np
import torch

from oracle import ecapa_oracle as EO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MODES = ("fp32", "3xf16", "tf32", "f16")


@functools.lru_cache(maxsize=None)
def audio():
    """tests/golden/*.wav resampled to 16 kHz on the library's kernels, and seeded signals: a chirp in noise of 1.3 s
    plus 37 samples, exactly 640 samples (5 frames), 3217 samples (21 frames, not a multiple of 16) and a tone with
    digital silence.  A list of float32 CPU tensors."""
    from scipy.io import wavfile

    from fastspeech2_b200.resample import Resampler
    out = []
    for name in ("sample_58k.wav", "sample_74k_waveglow.wav"):
        sr, w = wavfile.read(os.path.join(GOLDEN, name))
        x = torch.from_numpy((w / 32768.0).astype(np.float32))[None].cuda()
        y, n = Resampler(sr, 16000)(x, torch.tensor([x.shape[1]], device="cuda"))
        out.append(y[0, : int(n[0])].cpu())
    g = np.random.default_rng(5)
    t = np.arange(int(16000 * 1.3) + 37) / 16000.0
    out.append(torch.from_numpy((0.3 * np.sin(2 * np.pi * (200 * t + 900 * t * t)) + 0.05 * g.standard_normal(t.size)).astype(np.float32)))
    out.append(torch.from_numpy((0.2 * g.standard_normal(640)).astype(np.float32)))
    out.append(torch.from_numpy((0.1 * g.standard_normal(3217)).astype(np.float32)))
    tone = 0.25 * np.sin(2 * np.pi * 440 * np.arange(9000) / 16000.0)
    tone[3000:6000] = 0.0
    out.append(torch.from_numpy(tone.astype(np.float32)))
    return out


@functools.lru_cache(maxsize=None)
def model(C=1024, seed=0):
    """A seeded ECAPA_TDNN of width C with every BatchNorm's statistics from a float64 pass over audio()."""
    kw = {} if C == 1024 else {"channels": (C, C, C, C, 3 * C)}
    m = EO.seeded(seed, **kw).cuda()
    EO.calibrate(m, [w.cuda().double() for w in audio()[:4]])
    return m.eval()


def reference(m, wav):
    """float64 embedding of one utterance (a 1-D tensor); m is left in float32."""
    with torch.no_grad():
        m64 = m.double()
        try:
            return m64.embed(wav.cuda().double())
        finally:
            m.float()


def padded(wavs, nan=False):
    """[B, Nmax] float32 on the GPU (NaN past each length when nan), lens [B] int64."""
    n = max(len(w) for w in wavs)
    x = torch.full((len(wavs), n), float("nan") if nan else 0.0)
    for b, w in enumerate(wavs):
        x[b, : len(w)] = w
    return x.cuda(), torch.tensor([len(w) for w in wavs], device="cuda")
