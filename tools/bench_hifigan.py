#!/usr/bin/env python
"""Batched HiFi-GAN vocoder on one H100 (`HiFiGANVocoder`), printed as one JSON line.  Writes nothing.

    python tools/bench_hifigan.py [--steps 1] [--rounds 3]

Workload: the mels and frame counts `synthesize` returns for the 64 LJSpeech phoneme sequences of
tests/golden/filelist64.npz (random-init weights: only the lengths matter for time), as tools/bench_vocoder.py uses.
  hifigan_{v1,v3}_{3xf16,f16}   one HiFiGANVocoder call on the whole ragged batch (seeded random weights);
  melgan_3xf16                  one MelGANVocoder call on the same batch, for context;
  oracle_{v1,v3}_eager          the oracle module (oracle/hifigan_oracle.py) in eager PyTorch on the same GPU, fp32 with
                                weight norm removed and torch's default backend flags, one call on the [1, 80, sum(olens)]
                                paragraph, as hifi-gan's inference.py runs a generator.
Rows report ms per batch, audio-seconds per second (sum(olens) * 256 / 22050 over the time) and TFLOP/s from the FLOP per
mel frame `HiFiGANVocoder.flops_per_frame` computes from the config.  Per stage: the device time of each MRF (its
resblocks and sums) from one torch.profiler pass, against its compute bound (3xf16: 3 x FLOP, f16: 1 x FLOP at 989 TFLOP/s
dense f16) and an HBM bound (per convolution: the producer reads fp32 rows and writes the operand, the GEMM reads the
operand and writes fp32 rows, plus the residual read; 3.35 TB/s).
The timed variants run in alternating windows of `--steps` calls, median of `--rounds` windows.  The card name, power
limit and max SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_per_utterance import alternate, card, median  # noqa: E402

F16_TFLOPS, HBM_TBS, SAMPLE_RATE = 989.0, 3.35, 22050


def max_sm_clock():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=20)
        return r.stdout.strip() or None
    except Exception:
        return None


def stage_profile(voc, mels, olens) -> list:
    """Device ms of each MRF of one call, by launch position (csrc/hifigan.cu): prep, mel operand, conv_pre, then per
    stage 2 upsampling kernels and the MRF's nk * G + max(nk - 2, 0) kernels, then the post kernel."""
    cfg = voc.config
    U, nk = len(cfg["upsample_rates"]), len(cfg["resblock_kernel_sizes"])
    per = nk * (12 if cfg["resblock"] == "1" else 4) + max(nk - 2, 0)
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad():
        voc(mels, olens)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            voc(mels, olens)
            torch.cuda.synchronize()
    ev = sorted([e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                 and ("hifigan" in e.name or "tap_gemm" in e.name)], key=lambda e: e.time_range.start)
    if len(ev) != voc.launches():
        return [None] * U
    out, i = [], 3
    for _ in range(U):
        out.append(sum(e.time_range.elapsed_us() for e in ev[i + 2: i + 2 + per]) * 1e-3)
        i += 2 + per
    return out


def stage_bounds(voc, frames: int, mode: str) -> list:
    """Per stage: (C, GFLOP, compute-bound ms, HBM-bound ms) of the MRF over `frames` mel frames."""
    cfg = voc.config
    e = 4 if mode == "3xf16" else 2            # operand bytes per element: hi + lo planes, or the hi plane
    convs, steps = (6, 3) if cfg["resblock"] == "1" else (2, 2)
    out, up = [], 1
    for i, u in enumerate(cfg["upsample_rates"]):
        up *= u
        c = cfg["upsample_initial_channel"] // 2 ** (i + 1)
        rows = frames * up
        flop = sum(2 * convs * c * c * k for k in cfg["resblock_kernel_sizes"]) * rows
        nk = len(cfg["resblock_kernel_sizes"])
        byts = nk * rows * c * (convs * (8 + 2 * e) + steps * 4) + max(nk - 2, 0) * rows * c * 12
        out.append((c, flop * 1e-9, flop * (3 if mode == "3xf16" else 1) / (F16_TFLOPS * 1e12) * 1e3, byts / (HBM_TBS * 1e12) * 1e3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.hifigan import CONFIGS, HOP, HiFiGANVocoder
    from fastspeech2_b200.hparams import load_hp
    from fastspeech2_b200.melgan import MelGANVocoder
    from oracle import hifigan_oracle as O
    from oracle.melgan_oracle import Generator as MelGANGenerator

    dev = torch.device("cuda", torch.cuda.current_device())
    model = FeedForwardTransformer(68, 80, load_hp(), precision="3xf16")
    model.load_state_dict(synthetic_state_dict(0), strict=True)
    model = model.to(dev).eval()
    fl = np.load(os.path.join(ROOT, "tests", "golden", "filelist64.npz"))
    with torch.no_grad():
        mels, olens, _ = model.synthesize(torch.from_numpy(fl["xs"]).to(dev), torch.from_numpy(fl["ilens"]).to(dev))
    del model
    ol = [int(v) for v in olens.tolist()]
    frames = sum(ol)
    audio_s = frames * HOP / SAMPLE_RATE
    paragraph = torch.cat([mels[b, :n] for b, n in enumerate(ol)], 0).T[None].contiguous()     # [1, 80, sum(olens)]

    fns, vocs, oracles = {}, {}, {}
    for name in ("v1", "v3"):
        torch.manual_seed(0)
        g = O.Generator(CONFIGS[name]).eval()
        for m in ("3xf16", "f16"):
            v = HiFiGANVocoder(name, math_mode=m)
            v.load_state_dict(g.state_dict())
            vocs[(name, m)] = v.to(dev).eval()
            fns[f"hifigan_{name}_{m}"] = (lambda v=vocs[(name, m)]: v(mels, olens))
        g.remove_weight_norm()
        oracles[name] = g.to(dev)
        fns[f"oracle_{name}_eager"] = (lambda g=oracles[name]: g(paragraph))
    torch.manual_seed(0)
    mg = MelGANVocoder(math_mode="3xf16")
    mg.load_state_dict(MelGANGenerator().state_dict())
    mg = mg.to(dev).eval()
    fns["melgan_3xf16"] = lambda: mg(mels, olens)

    ms = alternate(fns, args.steps, args.rounds)
    timing = {}
    for key, w in ms.items():
        t = median(w)
        timing[key] = {"ms_per_batch": t, "ms_windows": w, "audio_seconds_per_second": audio_s / (t * 1e-3)}
        if key.startswith(("hifigan", "oracle")):
            name = key.split("_")[1]
            fpf = vocs[(name, "3xf16")].flops_per_frame()
            timing[key]["tflops"] = fpf * frames / (t * 1e-3) / 1e12
    for name in ("v1", "v3"):
        timing[f"hifigan_{name}_3xf16"]["speedup_over_eager"] = timing[f"oracle_{name}_eager"]["ms_per_batch"] / timing[f"hifigan_{name}_3xf16"]["ms_per_batch"]
        timing[f"hifigan_{name}_f16"]["speedup_over_eager"] = timing[f"oracle_{name}_eager"]["ms_per_batch"] / timing[f"hifigan_{name}_f16"]["ms_per_batch"]
    flops = {name: {"flop_per_frame": vocs[(name, "3xf16")].flops_per_frame(),
                    "hand_count": {"v1": 0.61e9, "v3": 45e6}[name]} for name in ("v1", "v3")}
    stages = {}
    for (name, m), v in vocs.items():
        got = stage_profile(v, mels, olens)
        stages[f"{name}_{m}"] = [{"C": c, "measured_ms": t, "gflop": gf, "compute_bound_ms": cb, "hbm_bound_ms": hb}
                                 for t, (c, gf, cb, hb) in zip(got, stage_bounds(v, frames, m))]
    info = card()
    info["max_sm_clock"] = max_sm_clock()
    line = {
        "metric": "batched HiFi-GAN vocoder: log-mels of filelist64 (synthesize) -> audio", "card": info, "B": len(ol),
        "valid_frames": frames, "Lmax": int(mels.shape[1]), "audio_seconds": audio_s, "timing": timing, "flops": flops,
        "mrf_stages": stages, "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32,
        "timing_note": f"eager launches, alternating windows of {args.steps} calls, median of {args.rounds} windows; stage bounds "
                       "count the valid rows only (sum(olens) * up_s), which is what the GEMMs run: dead tiles are skipped",
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
