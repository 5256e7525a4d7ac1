#!/usr/bin/env python
"""Batched vocoders on one H100 (`GriffinLimVocoder`, `MelGANVocoder`), printed as one JSON line.  Writes nothing.

    python tools/bench_vocoder.py [--iters 30] [--steps 2] [--rounds 3]

Workload: the mels and frame counts `synthesize` returns for the 64 LJSpeech phoneme sequences of
tests/golden/filelist64.npz (random-init weights: only the lengths matter for time), n_iters = 30 as in the reference.
  batched_3xf16 / batched_f16   one GriffinLimVocoder call on the whole ragged batch;
  looped_existing              the existing path on identical magnitudes: `mel_to_magnitude`, then `vocoder.griffin_lim`
                               (STFT class, 3xf16) called once per utterance on its own frames, same iterations;
  convergence                  spectral convergence ||STFT(y)| - M| / |M| over the batch after 10 and 30 iterations,
                               momentum 0 (the reference's algorithm) against 0.99 (fast Griffin-Lim), seed 0;
  melgan_3xf16 / melgan_f16    one MelGANVocoder call on the whole ragged batch (seeded random weights);
  melgan_oracle_eager          the CPU oracle's module (oracle/melgan_oracle.py) in eager PyTorch on the GPU, used as
                               inference.py uses the hub object (weight norm removed by eval(inference=True)): one
                               `inference` call on the [1, 80, sum(olens)] paragraph.
MelGAN rows also report TFLOP/s from 90.3 MFLOP per mel frame (counted over olens + 10 tail frames per utterance) and,
from one torch.profiler pass per mode, the fused ResStack kernels' device time per stage against the compute bound
(3xf16: 3 x FLOP, f16: 1 x FLOP at 989 TFLOP/s dense f16) and the HBM bound (each block reads x and writes x' once in
fp32, 3.35 TB/s).
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


MELGAN_MFLOP_PER_FRAME = 90.3
MELGAN_STAGES = ((256, 8), (128, 64), (64, 128), (32, 256))      # ResStack channels, rows per mel frame
F16_TFLOPS, HBM_TBS = 989.0, 3.35


def melgan_resstack_profile(voc, mels, olens) -> list:
    """Device ms of the ResStack kernels of one call, per stage, by launch position: prep, first-conv operand and GEMM,
    then per stage 2 upsampling kernels and the ResStack's kernels (3 fused blocks in f16 / 3xf16, 12 unfused kernels in
    fp32 / tf32), then the last conv (csrc/melgan.cu)."""
    per = [3 if fused(voc.math_mode, c) else 12 for c, _ in MELGAN_STAGES]
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad():
        voc(mels, olens)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            voc(mels, olens)
            torch.cuda.synchronize()
    ev = sorted([e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                 and ("melgan" in e.name or "tap_gemm" in e.name)], key=lambda e: e.time_range.start)
    if len(ev) != 3 + 8 + sum(per) + 1:
        return [None] * 4
    out, i = [], 3
    for n in per:
        out.append(sum(e.time_range.elapsed_us() for e in ev[i + 2: i + 2 + n]) * 1e-3)
        i += 2 + n
    return out


def fused(mode: str, c: int) -> bool:
    """csrc/melgan.cu fused_blocks(): the ResStacks that run as one fused kernel per block."""
    return (mode == "f16" and c <= 128) or (mode == "3xf16" and c <= 64)


def melgan_bounds(frames: int, mode: str) -> list:
    """Per stage: (GFLOP, compute-bound ms, HBM-bound ms) of the three residual blocks over `frames` mel frames, for the
    route the stage takes."""
    e = 4 if mode == "3xf16" else 2          # operand bytes per element: hi + lo planes, or the hi plane
    out = []
    for c, up in MELGAN_STAGES:
        rows = frames * up
        flop = 3 * rows * (2 * 3 * c * c + 2 * 2 * c * c)
        if fused(mode, c):
            byts = 3 * rows * 8 * c                 # per block: x read once (fp32), x' written once (fp32)
        else:
            byts = 3 * rows * (20 * c + 10 * c * e)  # taps, GEMM 3C, concat, GEMM 2C: fp32 activations + operands
        out.append((flop * 1e-9, flop * (3 if mode == "3xf16" else 1) / (F16_TFLOPS * 1e12) * 1e3, byts / (HBM_TBS * 1e12) * 1e3))
    return out


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
    from fastspeech2_b200.melgan import MelGANVocoder
    from fastspeech2_b200.vocoder import STFT, GriffinLimVocoder, griffin_lim
    from oracle.melgan_oracle import Generator

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

    torch.manual_seed(0)
    gen = Generator().eval()
    mg = {}
    for m in ("3xf16", "f16"):
        mg[m] = MelGANVocoder(math_mode=m)
        mg[m].load_state_dict(gen.state_dict())
        mg[m] = mg[m].to(dev).eval()
    gen = gen.eval(inference=True).to(dev)      # weight norm removed, as the hub object inference.py uses holds it
    paragraph = torch.cat([mels[b, :n] for b, n in enumerate(ol)], 0).T[None].contiguous()     # [1, 80, sum(olens)]
    fns = {"batched_3xf16": lambda: voc["3xf16"](mels, olens, n_iters=args.iters),
           "batched_f16": lambda: voc["f16"](mels, olens, n_iters=args.iters),
           "looped_existing": looped,
           "melgan_3xf16": lambda: mg["3xf16"](mels, olens),
           "melgan_f16": lambda: mg["f16"](mels, olens),
           "melgan_oracle_eager": lambda: gen.inference(paragraph)}
    ms = alternate(fns, args.steps, args.rounds)
    timing = {}
    for name, w in ms.items():
        t = median(w)
        timing[name] = {"ms_per_batch": t, "ms_windows": w, "audio_seconds_per_second": audio_s / (t * 1e-3)}
    timing["batched_3xf16_speedup_over_looped"] = timing["looped_existing"]["ms_per_batch"] / timing["batched_3xf16"]["ms_per_batch"]
    mel_audio_s = sum(n * hop for n in ol) / sr
    net_frames = {"melgan_3xf16": sum(ol) + 10 * len(ol), "melgan_f16": sum(ol) + 10 * len(ol), "melgan_oracle_eager": sum(ol) + 10}
    for name, fr in net_frames.items():
        t = timing[name]["ms_per_batch"]
        timing[name]["audio_seconds_per_second"] = mel_audio_s / (t * 1e-3)
        timing[name]["tflops"] = fr * MELGAN_MFLOP_PER_FRAME * 1e6 / (t * 1e-3) / 1e12
    resstack = {}
    for m in ("3xf16", "f16"):
        got = melgan_resstack_profile(mg[m], mels, olens)
        resstack[m] = [{"C": c, "fused": fused(m, c), "measured_ms": ms, "gflop": b[0], "compute_bound_ms": b[1], "hbm_bound_ms": b[2]}
                       for (c, _), ms, b in zip(MELGAN_STAGES, got, melgan_bounds(net_frames["melgan_3xf16"], m))]

    conv = {}
    for momentum in (0.0, 0.99):
        for it in (10, 30):
            audio, alens = voc["3xf16"](mels, olens, n_iters=it, momentum=momentum, seed=0)
            conv[f"momentum={momentum} iters={it}"] = spectral_convergence(stft, audio, alens, M, ol)
    line = {
        "metric": "batched Griffin-Lim vocoder: log-mels of filelist64 (synthesize) -> audio", "card": card(), "B": len(ol),
        "valid_frames": sum(ol), "Lmax": int(mels.shape[1]), "audio_seconds": audio_s, "n_iters": args.iters,
        "peak_magnitude": float(M.max()), "timing": timing, "spectral_convergence": conv, "melgan_resstack": resstack,
        "melgan_audio_seconds": mel_audio_s,
        "timing_note": f"eager launches, alternating windows of {args.steps} calls, median of {args.rounds} windows",
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
