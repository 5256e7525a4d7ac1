#!/usr/bin/env python
"""Batched BigVGAN vocoder on one H100 (`BigVGANVocoder`), printed as one JSON line.  Writes nothing.

    python tools/bench_bigvgan.py [--steps 1] [--rounds 3]

Workload: the mels and frame counts `synthesize` returns for the 64 LJSpeech phoneme sequences of
tests/golden/filelist64.npz (seeded random weights: only the lengths matter for time), as tools/bench_hifigan.py uses.
  bigvgan_{base,large}_{3xf16,f16}  one BigVGANVocoder call on the whole ragged batch (base_22khz_80band, 22khz_80band);
  oracle_{base,large}_eager          the oracle module (oracle/bigvgan_oracle.py) in eager PyTorch on the same GPU, fp32
                                     with weight norm removed and torch's default backend flags, one call on the
                                     [1, 80, sum(olens)] paragraph;
  window_base_3xf16_n32              time to the first audio (one `window` of 32 frames at start 0) and the whole
                                     `stream(chunk_frames=32)`.
Rows report ms per batch, audio-seconds per second (sum(olens) * 256 / 22050 over the time) and TFLOP/s from
`BigVGANVocoder.flops_per_frame`.  Per stage: the device time of one activation producer launch (bigvgan_act_kernel) from
one torch.profiler pass, against its HBM bound (it reads the valid rows' fp32 values once and writes every row of the
operand; 3.35 TB/s).  The timed variants run in alternating windows of `--steps` calls, median of `--rounds` windows.  The
card name, power limit and max SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_hifigan import HBM_TBS, SAMPLE_RATE, max_sm_clock  # noqa: E402
from bench_per_utterance import alternate, card, median  # noqa: E402

NAMES = {"base": "base_22khz_80band", "large": "22khz_80band"}


def act_profile(voc, mels, olens, mode: str) -> list:
    """Per stage s: (C'_s, launches, mean device us of one bigvgan_act_kernel launch, HBM-bound us of one launch), the
    stage found by launch position: the plain-rows producer (hifigan_act_kernel without lrelu, the generator chain's) opens
    conv_pre (first) and every upsampling."""
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad():
        voc(mels, olens)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            voc(mels, olens)
            torch.cuda.synchronize()
    ev = sorted([e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                 and ("bigvgan" in e.name or "hifigan_act_kernel" in e.name)],
                key=lambda e: e.time_range.start)
    cfg = voc.config
    U = len(cfg["upsample_rates"])
    per = [[] for _ in range(U)]
    s = -2
    for e in ev:
        if "hifigan_act_kernel" in e.name:
            s += 1
        elif "bigvgan_act_kernel" in e.name and 0 <= s < U:
            per[s].append(e.time_range.elapsed_us())
    out, up = [], 1
    valid, rows = int(olens.sum()), olens.numel() * mels.shape[1]
    ob = {"3xf16": 4, "f16": 2}.get(mode, 4)                           # operand bytes per element
    for i, u in enumerate(cfg["upsample_rates"]):
        up *= u
        c = (cfg["upsample_initial_channel"] // 2 ** (i + 1) + 31) // 32 * 32
        byts = valid * up * c * 4 + rows * up * c * ob
        t = sum(per[i]) / len(per[i]) if per[i] else None
        out.append({"C_padded": c, "launches": len(per[i]), "us_per_launch": t, "hbm_bound_us": byts / (HBM_TBS * 1e12) * 1e6})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.bigvgan import CONFIGS, HOP, BigVGANVocoder
    from fastspeech2_b200.hparams import load_hp
    from oracle import bigvgan_oracle as O

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

    fns, vocs = {}, {}
    for key, name in NAMES.items():
        torch.manual_seed(0)
        g = O.Generator(CONFIGS[name]).eval()
        for m in ("3xf16", "f16"):
            v = BigVGANVocoder(name, math_mode=m)
            v.load_state_dict(g.state_dict())
            vocs[(key, m)] = v.to(dev).eval()
            fns[f"bigvgan_{key}_{m}"] = (lambda v=vocs[(key, m)]: v(mels, olens))
        g.remove_weight_norm()
        g = g.to(dev)
        fns[f"oracle_{key}_eager"] = (lambda g=g: g(paragraph))

    with torch.no_grad():
        ms = alternate(fns, args.steps, args.rounds)
    timing = {}
    for k, w in ms.items():
        t = median(w)
        key = k.split("_")[1]
        timing[k] = {"ms_per_batch": t, "ms_windows": w, "audio_seconds_per_second": audio_s / (t * 1e-3),
                     "tflops": vocs[(key, "3xf16")].flops_per_frame() * frames / (t * 1e-3) / 1e12}
    for key in NAMES:
        for m in ("3xf16", "f16"):
            timing[f"bigvgan_{key}_{m}"]["speedup_over_eager"] = timing[f"oracle_{key}_eager"]["ms_per_batch"] / timing[f"bigvgan_{key}_{m}"]["ms_per_batch"]

    v = vocs[("base", "3xf16")]
    first, full = [], []
    with torch.no_grad():
        for r in range(args.rounds + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            v.window(mels, olens, 0, 32)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            for _ in v.stream(mels, olens, 32):
                pass
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            if r:                                                       # the first round warms the window workspace
                first.append((t1 - t0) * 1e3)
                full.append((t2 - t1) * 1e3)
    timing["window_base_3xf16_n32"] = {"first_audio_ms": median(first), "full_stream_ms": median(full), "first_audio_windows": first,
                                       "full_stream_windows": full}

    stages = {f"{key}_{m}": act_profile(vocs[(key, m)], mels, olens, m) for key, m in vocs}
    info = card()
    info["max_sm_clock"] = max_sm_clock()
    line = {
        "metric": "batched BigVGAN vocoder: log-mels of filelist64 (synthesize) -> audio", "card": info, "B": len(ol),
        "valid_frames": frames, "Lmax": int(mels.shape[1]), "audio_seconds": audio_s, "timing": timing,
        "flop_per_frame": {key: vocs[(key, "3xf16")].flops_per_frame() for key in NAMES}, "act_producer": stages,
        "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32,
        "timing_note": f"eager launches, alternating windows of {args.steps} calls, median of {args.rounds} windows",
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
