#!/usr/bin/env python
"""Batched Griffin-Lim vocoder (`GriffinLimVocoder`) on one H100, printed as one JSON line.  Writes nothing.

    python tools/bench_vocoder.py [--iters 30] [--steps 2] [--rounds 3]

Workload: the mels and frame counts `synthesize` returns for the 64 LJSpeech phoneme sequences of
tests/golden/filelist64.npz (random-init weights: only the lengths matter for time), n_iters = 30 as in the reference.
  batched_3xf16 / batched_f16   one GriffinLimVocoder call on the whole ragged batch;
  looped_existing              the existing path on identical magnitudes: `mel_to_magnitude`, then `vocoder.griffin_lim`
                               (STFT class, 3xf16) called once per utterance on its own frames, same iterations;
  convergence                  spectral convergence ||STFT(y)| - M| / |M| over the batch after 10 and 30 iterations,
                               momentum 0 (the reference's algorithm) against 0.99 (fast Griffin-Lim), seed 0.
The timed variants run in alternating windows of `--steps` calls, median of `--rounds` windows; audio-seconds per second
counts the valid samples, sum((olens - 1) * hop) / sample_rate.  The card name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_per_utterance import alternate, card, median  # noqa: E402


def spectral_convergence(stft, audio, alens, M, olens) -> float:
    num = den = 0.0
    for b in range(audio.shape[0]):
        n = int(olens[b])
        mag, _ = stft.transform(audio[b: b + 1, : int(alens[b])])
        num += float((mag[0, :, :n] - M[b, :, :n]).pow(2).sum())
        den += float(M[b, :, :n].pow(2).sum())
    return (num / den) ** 0.5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.hparams import load_hp
    from fastspeech2_b200.vocoder import STFT, GriffinLimVocoder, griffin_lim

    dev = torch.device("cuda", torch.cuda.current_device())
    hp = load_hp()
    model = FeedForwardTransformer(68, 80, hp, precision="3xf16")
    model.load_state_dict(synthetic_state_dict(0), strict=True)
    model = model.to(dev).eval()
    fl = np.load(os.path.join(ROOT, "tests", "golden", "filelist64.npz"))
    with torch.no_grad():
        mels, olens, _ = model.synthesize(torch.from_numpy(fl["xs"]).to(dev), torch.from_numpy(fl["ilens"]).to(dev))
    voc = {m: GriffinLimVocoder.from_hp(hp, math_mode=m).to(dev) for m in ("3xf16", "f16")}
    hop, sr = voc["3xf16"].hop_length, voc["3xf16"].sample_rate
    ol = [int(v) for v in olens.tolist()]
    audio_s = sum((n - 1) * hop for n in ol) / sr
    M = voc["3xf16"].mel_to_magnitude(mels, olens)
    stft = STFT(voc["3xf16"].n_fft, hop, voc["3xf16"].win_length, math_mode="3xf16").to(dev)
    angles = [torch.zeros(1, M.shape[1], n, device=dev) for n in ol]

    def looped():
        return [griffin_lim(M[b: b + 1, :, :n], stft, args.iters, angles=angles[b]) for b, n in enumerate(ol)]

    fns = {"batched_3xf16": lambda: voc["3xf16"](mels, olens, n_iters=args.iters),
           "batched_f16": lambda: voc["f16"](mels, olens, n_iters=args.iters),
           "looped_existing": looped}
    ms = alternate(fns, args.steps, args.rounds)
    timing = {}
    for name, w in ms.items():
        t = median(w)
        timing[name] = {"ms_per_batch": t, "ms_windows": w, "audio_seconds_per_second": audio_s / (t * 1e-3)}
    timing["batched_3xf16_speedup_over_looped"] = timing["looped_existing"]["ms_per_batch"] / timing["batched_3xf16"]["ms_per_batch"]

    conv = {}
    for momentum in (0.0, 0.99):
        for it in (10, 30):
            audio, alens = voc["3xf16"](mels, olens, n_iters=it, momentum=momentum, seed=0)
            conv[f"momentum={momentum} iters={it}"] = spectral_convergence(stft, audio, alens, M, ol)
    line = {
        "metric": "batched Griffin-Lim vocoder: log-mels of filelist64 (synthesize) -> audio", "card": card(), "B": len(ol),
        "valid_frames": sum(ol), "Lmax": int(mels.shape[1]), "audio_seconds": audio_s, "n_iters": args.iters,
        "peak_magnitude": float(M.max()), "timing": timing, "spectral_convergence": conv,
        "timing_note": f"eager launches, alternating windows of {args.steps} calls, median of {args.rounds} windows",
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
