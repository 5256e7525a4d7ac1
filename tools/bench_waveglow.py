#!/usr/bin/env python
"""Batched WaveGlow vocoder on one H100 (`WaveGlowVocoder`), printed as one JSON line.  Writes nothing.

    python tools/bench_waveglow.py [--steps 1] [--rounds 3] [--channels 256,512]

Workload: the mels and frame counts `synthesize` returns for the 64 LJSpeech phoneme sequences of
tests/golden/filelist64.npz (random-init FastSpeech2 weights: only the lengths matter for time), vocoded with seeded
random WaveGlow weights at n_channels C = 256 and 512:
  waveglow_C{C}_3xf16 / _f16   one WaveGlowVocoder call on the whole ragged batch (sigma 0.6, seed 0);
  oracle_C{C}_eager_fp32 / _fp16  the oracle's module (oracle/waveglow_oracle.py) in eager PyTorch on the same GPU, weight
                               norm removed, as the reference's notebook uses the hub object: one `infer` call on the
                               [1, 80, sum(olens)] paragraph (fp32: torch's defaults, so cuDNN may use TF32; fp16:
                               `.half()` module and input).  If a call runs out of memory it runs per utterance instead,
                               and the row says so.
Each row reports audio-seconds per second (sum(olens) * 256 / 22050 over the call time) and TFLOP/s from the shapes:
126 C^2 + 20480 C FLOP per step and flow, x 12 flows x 32 steps per mel frame, plus 13.1 MFLOP per frame for the
upsampling (16.7 GFLOP per frame at C = 512, 5.18 at C = 256).  One torch.profiler pass per batched row gives the device
time per kernel class (upsampling, start, cond GEMM, in-layer GEMM, gate, res_skip GEMM, flow kernel) against its compute
bound (FLOP x 3 in 3xf16, x 1 in f16, at 989 TFLOP/s dense f16) and its HBM bound (the bytes each class must move once,
at 3.35 TB/s).  Each variant runs `--rounds` windows of `--steps` calls after a warm-up call (median window); variants run one after
another, since at C = 512 the batched call's workspace alone is tens of GB.  The card
name and power limit are read in the same run.
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

F16_TFLOPS, HBM_TBS, SR = 989.0, 3.35, 22050
UP_FLOP_PER_FRAME = 2 * 320 * 80 * 256


def flop_per_frame(C: int) -> float:
    return (126 * C * C + 20480 * C) * 12 * 32 + UP_FLOP_PER_FRAME


def class_flop_bytes(C: int, frames: int, x3: bool) -> dict:
    """Per call: (FLOP, bytes each kernel class moves at least once: operands at the width read, fp32 rows)."""
    e = 4 if x3 else 2                                  # bytes per operand element: hi + lo planes, or the hi plane
    rows = 12 * 32 * frames                             # step rows, summed over the 12 flows
    return {
        "upsampling": (2.0 * frames * 320 * 20480, frames * 320 * 4 + 32 * frames * 640 * (4 + 4 + e)),
        "start": (0.0, rows * C * (4 + e)),
        "cond_gemm": (rows * 8 * 2.0 * 640 * 2 * C, rows * 8 * (640 * e + 2 * C * 4)),
        "in_layer_gemm": (rows * 8 * 2.0 * 3 * C * 2 * C, rows * 8 * (C * e + 2 * 2 * C * 4)),
        "gate": (0.0, rows * (8 * (2 * C * 4 + C * e) + 7 * C * 4)),
        "res_skip_gemm": (rows * (7 * 2.0 * C * 2 * C + 2.0 * C * C), rows * (7 * (C * e + 2 * C * 4 + C * e) + 8 * (C * e + 2 * C * 4))),
        "flow": (rows * 2.0 * 8 * C, rows * C * 4),
    }


def profile_classes(voc, mels, olens) -> dict:
    """Device ms per kernel class of one call, from the kernel sequence of csrc/waveglow.cu: prep, noise, up operand,
    up GEMM, (cond planes,) then per flow start, 8 x (cond GEMM, in-layer GEMM, gate, res GEMM (layers 0-6), skip GEMM),
    the flow kernel."""
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad():
        voc(mels, olens, sigma=0.6, seed=0)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            voc(mels, olens, sigma=0.6, seed=0)
            torch.cuda.synchronize()
    evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
                  and "Memset" not in e.name), key=lambda e: e.time_range.start)
    out = {k: 0.0 for k in ("upsampling", "start", "cond_gemm", "in_layer_gemm", "gate", "res_skip_gemm", "flow")}
    state, layer, after_gate = "up", 0, 0
    for e in evs:
        n, ms = e.name, e.device_time / 1e3 if hasattr(e, "device_time") else e.cuda_time / 1e3
        gemm = "tap_gemm" in n
        if "wg_start" in n:
            state, layer = "cond", 0
            out["start"] += ms
        elif "wg_gate" in n:
            out["gate"] += ms
            state, after_gate = "res_skip", (2 if layer < 7 else 1)
        elif "wg_flow" in n:
            out["flow"] += ms
        elif gemm and state == "cond":
            out["cond_gemm"] += ms
            state = "in"
        elif gemm and state == "in":
            out["in_layer_gemm"] += ms
        elif gemm and state == "res_skip":
            out["res_skip_gemm"] += ms
            after_gate -= 1
            if after_gate == 0:
                state, layer = "cond", layer + 1
        else:                                           # prep, noise, up operand, up GEMM, cond planes
            out["upsampling"] += ms
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--channels", default="256,512")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.hparams import load_hp
    from fastspeech2_b200.waveglow import WaveGlowVocoder
    from oracle import waveglow_oracle as O

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    model = FeedForwardTransformer(68, 80, load_hp())
    model.load_state_dict(synthetic_state_dict(0), strict=True)
    model = model.to(dev).eval()
    fl = np.load(os.path.join(ROOT, "tests", "golden", "filelist64.npz"))
    with torch.no_grad():
        mels, olens, _ = model.synthesize(torch.from_numpy(fl["xs"]).to(dev), torch.from_numpy(fl["ilens"]).to(dev))
    del model
    ol = [int(v) for v in olens.tolist()]
    frames = sum(ol)
    audio_s = frames * 256 / SR
    paragraph = torch.cat([mels[b, :n] for b, n in enumerate(ol)], 0).T[None].contiguous()     # [1, 80, sum(olens)]
    rows, profiles = {}, {}
    for C in [int(c) for c in args.channels.split(",")]:
        torch.manual_seed(C)
        g = O.WaveGlow(C)
        with torch.no_grad():
            for wn in g.WN:
                wn.end.weight.normal_(0, 1.0 / C ** 0.5)
                wn.end.bias.normal_(0, 0.1)
        voc = {}
        for m in ("3xf16", "f16"):
            v = WaveGlowVocoder(n_channels=C, math_mode=m)
            v.load_state_dict(g.state_dict())
            voc[m] = v.to(dev).eval()
        eager32 = O.WaveGlow.remove_weightnorm(g).to(dev).eval()
        eager16 = O.WaveGlow.remove_weightnorm(O.WaveGlow(C))
        eager16.load_state_dict(eager32.state_dict())
        eager16 = eager16.half().to(dev).eval()
        notes = {}

        def eager(mod, half):
            def run():
                x = paragraph.half() if half else paragraph
                try:
                    return mod.infer(x, 0.6)
                except torch.cuda.OutOfMemoryError:
                    notes[id(mod)] = "per utterance (the paragraph ran out of memory)"
                    torch.cuda.empty_cache()
                    return [mod.infer(mels[b: b + 1, :n].transpose(1, 2).contiguous().to(x.dtype), 0.6) for b, n in enumerate(ol)]
            return run

        # one variant at a time (warm-up call, then `rounds` windows of `steps` calls): at C = 512 a batched call's
        # workspace is tens of GB, so a vocoder frees its workspace before the next variant runs
        fns = {f"waveglow_C{C}_3xf16": ("3xf16", lambda v=voc["3xf16"]: v(mels, olens, sigma=0.6, seed=0)),
               f"waveglow_C{C}_f16": ("f16", lambda v=voc["f16"]: v(mels, olens, sigma=0.6, seed=0)),
               f"oracle_C{C}_eager_fp32": (None, eager(eager32, False)),
               f"oracle_C{C}_eager_fp16": (None, eager(eager16, True))}
        for name, (m, fn) in fns.items():
            v = alternate({name: fn}, args.steps, args.rounds)[name]
            t = median(v)
            row = {"ms": t, "ms_windows": v, "audio_s_per_s": audio_s / (t * 1e-3),
                   "tflops": flop_per_frame(C) * frames / (t * 1e-3) / 1e12}
            mod = eager32 if name.endswith("fp32") else eager16 if name.endswith("fp16") else None
            if mod is not None and id(mod) in notes:
                row["note"] = notes[id(mod)]
            if m is not None:
                got = profile_classes(voc[m], mels, olens)
                fb = class_flop_bytes(C, frames, m == "3xf16")
                profiles[f"C{C}_{m}"] = {k: {"ms": round(got[k], 3),
                                              "compute_bound_ms": round(fb[k][0] * (3 if m == "3xf16" else 1) / (F16_TFLOPS * 1e12) * 1e3, 3),
                                              "hbm_bound_ms": round(fb[k][1] / (HBM_TBS * 1e12) * 1e3, 3)} for k in got}
                row["workspace_gb"] = round(sum(w.numel() for w in voc[m]._ws.values()) / 1e9, 2)
                voc[m]._ws.clear()
            rows[name] = row
            torch.cuda.empty_cache()
        del voc, eager32, eager16, g
        torch.cuda.empty_cache()
    line = {"metric": "batched WaveGlow vocoder: log-mels of filelist64 (synthesize) -> audio", "card": card(), "B": len(ol),
            "Lmax": int(mels.shape[1]), "frames": frames, "audio_seconds": audio_s,
            "gflop_per_frame": {f"C{c}": flop_per_frame(int(c)) / 1e9 for c in args.channels.split(",")},
            "rows": rows, "profile": profiles}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
