#!/usr/bin/env python
"""Training-feature extraction on one H100 (`FeatureExtractor`, `python -m fastspeech2_b200.preprocess`), printed as one
JSON line.  Writes nothing in the tree (the command's files go to a temporary directory).

    python tools/bench_features.py [--steps 5] [--rounds 3]

Workload: the 64 utterances of tests/golden/filelist64.npz at olens[b] * hop samples (about 423 s at 22.05 kHz), filled
with a seeded speech-like signal (harmonics of a moving F0, a slow envelope and a little noise).
  mel_energy / pitch   one call on the whole ragged batch (3xf16 for the GEMMs; DIO is float64), device events around
                       `--steps` calls, median of `--rounds` windows; audio-seconds per second, and the work counted
                       from shapes: 2 * rows * n_fft * cpad + 2 * rows * mpad * n_mels for the two GEMMs (rows = the valid
                       frames), and 2 * (883 + sum of the 4h Nuttall taps) float64 flop per sample for DIO's filters.
  oracle_numpy         the float64 numpy restatement (oracle/dio_oracle.py) on the same batch on the CPU, for context:
                       numpy, not pyworld, whose time is not measured here.
  command              wall time of the preprocessing command on a directory of the 64 utterances as int16 wav files,
                       beside the time to read them alone, to show which of the two bounds it.
The card name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_per_utterance import card, median  # noqa: E402

HOP, FS = 256, 22050


def speechlike(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / FS
    f0 = 120 + 60 * np.sin(2 * np.pi * 0.7 * t + seed) + 20 * np.sin(2 * np.pi * 2.3 * t)
    ph = 2 * np.pi * np.cumsum(f0) / FS
    x = sum((0.25 / k) * np.sin(k * ph + k * seed) for k in range(1, 8))
    env = 0.6 + 0.4 * np.sin(2 * np.pi * 1.1 * t + seed)
    return (x * env + 0.002 * rng.standard_normal(n)).astype(np.float32)


def timed(fn, steps, rounds):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / steps)
    return median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_features needs a CUDA device")
    from fastspeech2_b200.features import FeatureExtractor
    from fastspeech2_b200.hparams import load_hp
    from fastspeech2_b200.preprocess import read_wav_np, run
    from oracle import dio_oracle as D

    olens = np.load(os.path.join(ROOT, "tests", "golden", "filelist64.npz"))["olens"].astype(np.int64)
    n = [int(v) * HOP for v in olens]
    xs = [speechlike(k, i) for i, k in enumerate(n)]
    audio_s = sum(n) / FS
    w = torch.zeros(len(n), max(n))
    for b, x in enumerate(xs):
        w[b, : n[b]] = torch.from_numpy(x)
    w, L = w.cuda(), torch.tensor(n).cuda()
    fx = FeatureExtractor().cuda()
    res = {"metric": "features", "card": card(), "utterances": len(n), "audio_s": round(audio_s, 1)}

    rows = sum(k // HOP + 1 for k in n)
    gemm_flop = 2.0 * rows * (1024 * 1088 + 576 * 80)                    # forward DFT, then the mel filterbank
    boundary = D.band_edges()
    taps = 883 + sum(4 * D.matlab_round(FS / b / 2.0) for b in boundary)
    dio_flop = 2.0 * taps * sum(k + 1 for k in n)
    for name, fn, flop in (("mel_energy", lambda: fx.mel_energy(w, L), gemm_flop), ("pitch", lambda: fx.pitch(w, L), dio_flop)):
        ms = timed(fn, args.steps, args.rounds)
        res[name] = {"ms": round(ms, 3), "audio_s_per_s": round(audio_s / ms * 1000, 0), "gflop": round(flop / 1e9, 2),
                     "tflop_per_s": round(flop / ms / 1e9, 2)}
    res["pitch"]["fp64_taps_per_sample"] = taps

    t0 = time.perf_counter()
    for x in xs:
        D.dio(x.astype(np.float64), FS, frame_period=D.frame_period_ms(HOP, FS))
    t1 = time.perf_counter()
    for x in xs:
        D.mel_energy(x)
    t2 = time.perf_counter()
    res["oracle_numpy"] = {"pitch_s": round(t1 - t0, 2), "mel_energy_s": round(t2 - t1, 2),
                           "note": "float64 numpy restatement on the CPU, not pyworld"}

    from scipy.io import wavfile
    with tempfile.TemporaryDirectory() as tmp:
        wd = os.path.join(tmp, "wavs")
        os.makedirs(wd)
        for i, x in enumerate(xs):
            wavfile.write(os.path.join(wd, f"u{i:03d}.wav"), FS, np.round(x * 32767).astype(np.int16))
        t0 = time.perf_counter()
        for f in sorted(os.listdir(wd)):
            read_wav_np(os.path.join(wd, f), FS)
        t_read = time.perf_counter() - t0
        hp = load_hp()
        run(wd, hp, os.path.join(tmp, "warm"), log=lambda *a: None)          # untimed: first-use costs (module load, context)
        t0 = time.perf_counter()
        run(wd, hp, os.path.join(tmp, "out"), stats=True, log=lambda *a: None)
        t_cmd = time.perf_counter() - t0
    res["command"] = {"wall_s": round(t_cmd, 3), "read_wavs_s": round(t_read, 3),
                      "gpu_s": round((res["mel_energy"]["ms"] + res["pitch"]["ms"]) / 1000, 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
