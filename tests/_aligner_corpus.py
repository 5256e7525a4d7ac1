"""Synthetic aligner corpus from tests/golden/align_filelist.npz (LJSpeech phoneme strings and MFA durations): each
phoneme token is a seeded 80-d log-mel-like prototype, held with noise for its MFA duration.  The true durations are the
MFA ones, so an aligner trained on it can be scored against them (tests/test_gpu_aligner.py, tools/bench_aligner.py)."""
import os

import numpy as np

from fastspeech2_b200 import aligner as A

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def fixture_lines(n=None):
    """Lines (text empty, durations = MFA) of the first n fixture utterances."""
    z = np.load(os.path.join(GOLDEN, "align_filelist.npz"))
    off, dur = z["offsets"], z["durations"].astype(np.int64)
    n = len(z["phonemes"]) if n is None else n
    return [A.Line("", None, dur[off[i]: off[i + 1]].tolist(), str(z["phonemes"][i]).split(), str(z["wavs"][i])) for i in range(n)]


def render(lines, seed=0, noise=0.5):
    """{id: mel [L, 80] float32}: token prototypes N(-5, 2) per channel, plus N(0, noise) per frame."""
    tokens = sorted({p for ln in lines for p in ln.phonemes})
    rng = np.random.default_rng(seed)
    proto = {t: rng.normal(-5.0, 2.0, 80) for t in tokens}
    out = {}
    for ln in lines:
        frames = np.concatenate([np.repeat(proto[p][None], d, 0) for p, d in zip(ln.phonemes, ln.durations)])
        out[ln.id] = (frames + rng.normal(0.0, noise, frames.shape)).astype(np.float32)
    return out
