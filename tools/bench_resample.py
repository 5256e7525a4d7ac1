#!/usr/bin/env python
"""Resampling on one H100 (`Resampler`, `python -m fastspeech2_b200.preprocess --resample`), printed as one JSON line.
Writes nothing in the tree (the preprocessing trees go to a temporary directory).

    python tools/bench_resample.py [--steps 5] [--rounds 3] [--oracle-utts 2] [--profile] [--corpus 32]

Workloads, seeded:
  down_48k   B = 64 LJSpeech-length utterances (1 to 10 s, uniform) at 48 kHz -> 22.05 kHz: a VCTK-style corpus
  up_48k     B = 64 vocoder-shaped batches at 22.05 kHz -> 48 kHz: olens U[150, 870] frames * 256 samples, as a
             server taking a vocoder's (audio, alens) to 48 kHz gets them
each as device events around `--steps` calls, median of `--rounds` windows: ms per batch and output samples/s.  `--profile`
adds, in a separate run, torch.profiler's device time of the clock pass (rs_clock_kernel) and the tap pass
(rs_taps_kernel).
  oracle     the float64 numpy restatement on the first `--oracle-utts` utterances on one CPU core, s per utterance, and
             whether the GPU matches it bit for bit there.
  preprocess `preprocess` end to end (host wall clock, a warm-up run first) on `--corpus` synthetic utterances written as
             int16 files at 48 kHz with --resample, against the same utterances at 22.05 kHz without it.
The card name, power limit and max SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_evaluate import timed  # noqa: E402
from bench_per_utterance import card, median  # noqa: E402

B, FS = 64, 22050


def max_sm_clock():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=20)
        return r.stdout.strip() or None
    except Exception:
        return None


def speech(n, seed, sr):
    """A gliding harmonic tone under a slow envelope plus a little noise, peak about 0.6."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    f0 = 120 + 50 * np.sin(2 * np.pi * 0.5 * t + seed)
    ph = 2 * np.pi * np.cumsum(f0) / sr
    x = sum((0.3 / k) * np.sin(k * ph) for k in range(1, 6)) * (0.6 + 0.3 * np.sin(2 * np.pi * 0.9 * t))
    return (x + 0.003 * rng.standard_normal(n)).astype(np.float32)


def workloads(seed=0):
    rng = np.random.default_rng(seed)
    secs = rng.uniform(1.0, 10.0, B)
    down = [speech(int(s * 48000), k, 48000) for k, s in enumerate(secs)]
    frames = rng.integers(150, 871, B)
    up = [speech(int(f) * 256, k, FS) for k, f in enumerate(frames)]
    return down, up


def pad(xs):
    n = [len(x) for x in xs]
    w = torch.zeros((len(xs), max(n)))
    for b, x in enumerate(xs):
        w[b, : n[b]] = torch.from_numpy(x)
    return w.cuda(), torch.tensor(n).cuda()


def corpus_run(n_utts, args):
    """preprocess wall time on a 48 kHz tree with --resample and on the 22.05 kHz tree, each after a warm-up run."""
    from scipy.io import wavfile

    from fastspeech2_b200.hparams import load_hp
    from fastspeech2_b200.preprocess import run
    rng = np.random.default_rng(3)
    secs = rng.uniform(1.0, 10.0, n_utts)
    hp = load_hp()
    out = {"utterances": n_utts, "audio_s": round(float(secs.sum()), 1)}
    with tempfile.TemporaryDirectory() as tmp:
        for sr in (48000, FS):
            d = os.path.join(tmp, str(sr))
            os.makedirs(d)
            for k, s in enumerate(secs):
                wavfile.write(os.path.join(d, f"u{k:04d}.wav"), sr, np.round(speech(int(s * sr), k, sr) * 32767).astype(np.int16))
        for sr, flag in ((48000, True), (FS, False)):
            d = os.path.join(tmp, str(sr))
            run(d, hp, os.path.join(tmp, "warm"), log=lambda *a: None, resample=flag)
            times = []
            for r in range(args.rounds):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                run(d, hp, os.path.join(tmp, f"out{sr}_{r}"), log=lambda *a: None, resample=flag)
                torch.cuda.synchronize()
                times.append(time.perf_counter() - t0)
            out["s_48k_resample" if flag else "s_22k_native"] = round(median(times), 3)
    out["resampling_adds"] = round(out["s_48k_resample"] / out["s_22k_native"] - 1, 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--oracle-utts", type=int, default=2)
    ap.add_argument("--corpus", type=int, default=32)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resample needs a CUDA device")
    from fastspeech2_b200.resample import Resampler, workspace_bytes
    from oracle import resample_oracle as R

    down, up = workloads()
    cases = {"down_48k": (48000, FS, down), "up_48k": (FS, 48000, up)}
    out = {"metric": "resampling, B = 64", "card": {**card(), "max_sm_clock": max_sm_clock()}, "B": B}
    calls = {}
    for name, (so, sn, xs) in cases.items():
        rs = Resampler(so, sn)
        w, n = pad(xs)
        calls[name] = (rs, w, n)
        y, ol = rs(w, n)
        samples = int(ol.sum())
        ms = timed(lambda: rs(w, n), args.steps, args.rounds)
        out[name] = {"orig_sr": so, "new_sr": sn, "Nmax": int(w.shape[1]), "output_samples": samples,
                     "workspace_bytes": workspace_bytes(B, w.shape[1], so, sn), "ms_per_batch": round(ms, 3),
                     "output_samples_per_s": float(f"{samples / ms * 1e3:.4g}")}
        k = args.oracle_utts
        y, ol = y.cpu().numpy(), ol.cpu().numpy()
        t0 = time.perf_counter()
        want = [R.resample(xs[b], so, sn) for b in range(k)]
        dt = time.perf_counter() - t0
        out[name]["oracle"] = {"utterances": k, "s_per_utt": round(dt / k, 3),
                               "output_samples_per_s": float(f"{sum(len(v) for v in want) / dt:.4g}"),
                               "bit_identical": bool(all(np.array_equal(y[b, : ol[b]].view(np.int32), want[b].view(np.int32))
                                                         for b in range(k)))}

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        per = {}
        for name, (rs, w, n) in calls.items():
            rs(w, n)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    rs(w, n)
                torch.cuda.synchronize()
            for e in prof.events():
                if e.device_type.name == "CUDA" and "rs_" in e.name:
                    k = e.name.split("rs_")[1].split("_kernel")[0]
                    per.setdefault(name, {}).setdefault(k, 0.0)
                    per[name][k] += e.device_time / 1e3 / args.steps
        out["kernel_ms"] = {c: {k: round(v, 3) for k, v in sorted(d.items())} for c, d in per.items()}

    if args.corpus:
        out["preprocess"] = corpus_run(args.corpus, args)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
