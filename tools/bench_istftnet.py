#!/usr/bin/env python
"""Batched iSTFTNet vocoder on one H100 (`ISTFTNetVocoder`) against HiFi-GAN V1 in the same process, printed as one JSON
line.  Writes nothing.

    python tools/bench_istftnet.py [--steps 1] [--rounds 3]

Workload: the mels and frame counts `synthesize` returns for the 64 LJSpeech phoneme sequences of
tests/golden/filelist64.npz (random-init weights: only the lengths matter for time), as tools/bench_hifigan.py uses.
  istftnet_v1_{3xf16,f16}   one ISTFTNetVocoder call (C8C8I) on the whole ragged batch;
  hifigan_v1_{3xf16,f16}    one HiFiGANVocoder V1 call on the same batch, alternated with the above;
  oracle_istftnet_eager     the oracle module (oracle/istftnet_oracle.py) in eager PyTorch on the same GPU, fp32 with weight
                            norm removed, one call on the [1, 80, sum(olens)] paragraph.
Rows report ms per batch and audio-seconds per second (sum(olens) * 256 / 22050 over the time).  first_audio_ms: one
`window(mels, olens, 0, 32)` call (the first 32 frames of every utterance), the latency to the first audio of a stream.
Per kernel: device time by kernel name from one torch.profiler pass per vocoder; for the head, its HBM bound (it reads the
last MRF's two fp32 buffers over the valid rows and writes the audio; 3.35 TB/s).  The timed variants run in alternating
windows of `--steps` calls, median of `--rounds` windows.  The card name, power limit and max SM clock are read in the
same run.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_hifigan import max_sm_clock  # noqa: E402
from bench_per_utterance import alternate, card, median  # noqa: E402

HBM_TBS, SAMPLE_RATE = 3.35, 22050


def kernel_profile(voc, mels, olens) -> dict:
    """Device ms per kernel name of one call."""
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad():
        voc(mels, olens)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            voc(mels, olens)
            torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            m = re.search(r"(\w+)(?:<[^(]*>)?\(", e.name)
            name = m.group(1) if m else e.name
            out[name] = out.get(name, 0.0) + e.time_range.elapsed_us() * 1e-3
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.hifigan import CONFIGS as HCONFIGS, HiFiGANVocoder
    from fastspeech2_b200.hparams import load_hp
    from fastspeech2_b200.istftnet import CONFIGS, HOP, ISTFTNetVocoder
    from oracle import hifigan_oracle as HO
    from oracle import istftnet_oracle as O

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

    torch.manual_seed(0)
    gi = O.Generator(CONFIGS["v1"]).eval()
    torch.manual_seed(0)
    gh = HO.Generator(HCONFIGS["v1"]).eval()
    fns, vocs = {}, {}
    for m in ("3xf16", "f16"):
        for key, cls, g in (("istftnet", ISTFTNetVocoder, gi), ("hifigan", HiFiGANVocoder, gh)):
            v = cls("v1", math_mode=m)
            v.load_state_dict(g.state_dict())
            vocs[(key, m)] = v.to(dev).eval()
            fns[f"{key}_v1_{m}"] = (lambda v=vocs[(key, m)]: v(mels, olens))
    gi.remove_weight_norm()
    gi = gi.to(dev)
    fns["oracle_istftnet_eager"] = lambda: gi(paragraph)
    for m in ("3xf16", "f16"):
        for key in ("istftnet", "hifigan"):
            fns[f"{key}_v1_{m}_first_audio"] = (lambda v=vocs[(key, m)]: v.window(mels, olens, 0, 32))

    ms = alternate(fns, args.steps, args.rounds)
    timing = {}
    for key, w in ms.items():
        t = median(w)
        timing[key] = {"ms": t, "ms_windows": w}
        if not key.endswith("first_audio"):
            timing[key]["audio_seconds_per_second"] = audio_s / (t * 1e-3)
    for m in ("3xf16", "f16"):
        timing[f"istftnet_v1_{m}"]["speedup_over_hifigan_v1"] = timing[f"hifigan_v1_{m}"]["ms"] / timing[f"istftnet_v1_{m}"]["ms"]
        timing[f"istftnet_v1_{m}"]["speedup_over_eager"] = timing["oracle_istftnet_eager"]["ms"] / timing[f"istftnet_v1_{m}"]["ms"]
    kernels = {f"{k}_{m}": kernel_profile(v, mels, olens) for (k, m), v in vocs.items()}
    rows = frames * 64                                   # the head's valid last-level rows
    head_bytes = 2 * rows * 128 * 4 + frames * HOP * 4
    head = {"bytes": head_bytes, "hbm_bound_ms": head_bytes / (HBM_TBS * 1e12) * 1e3,
            "measured_ms": {m: kernels[f"istftnet_{m}"].get("istftnet_head_kernel") for m in ("3xf16", "f16")},
            "conv_post_gflop": rows * 128 * 18 * 7 * 2 * 1e-9}
    flops = {"istftnet_v1": vocs[("istftnet", "3xf16")].flops_per_frame(), "hifigan_v1": vocs[("hifigan", "3xf16")].flops_per_frame()}
    info = card()
    info["max_sm_clock"] = max_sm_clock()
    line = {
        "metric": "batched iSTFTNet (C8C8I) vs HiFi-GAN V1 vocoder: log-mels of filelist64 (synthesize) -> audio", "card": info,
        "B": len(ol), "valid_frames": frames, "Lmax": int(mels.shape[1]), "audio_seconds": audio_s, "timing": timing,
        "flop_per_frame": flops, "head": head, "kernels_ms": kernels,
        "timing_note": f"eager launches, alternating windows of {args.steps} calls, median of {args.rounds} windows",
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
