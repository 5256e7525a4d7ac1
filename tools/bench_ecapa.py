"""Throughput of the ECAPA-TDNN speaker encoder (DESIGN.md section 28) on a 64-utterance batch of LJSpeech-like durations
(1-10 s, seeded), against SpeechBrain's network restated in torch (oracle/ecapa_oracle.py) in fp32 on the same GPU: one
utterance at a time (how ESPnet's extractor loops over a corpus) and padded-batched.  Arms alternate.  Prints one JSON line
with the card's name and power limit, audio-seconds per second and whole-program TFLOP/s from the FLOPs the shapes imply.

    python tools/bench_ecapa.py [--reps 5] [--modes 3xf16,f16,fp32,tf32]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fastspeech2_b200.ecapa import ECAPAEncoder  # noqa: E402
from oracle import ecapa_oracle as EO  # noqa: E402


def flops_per_frame(a):
    """Multiply-adds x 2 per frame of every convolution GEMM (the per-utterance vectors and the front end are not counted)."""
    C, nm, M, A, s = a["channels"], a["n_mels"], a["mfa_channels"], a["attention_channels"], a["scale"]
    c8 = C // s
    macs = a["kernel_sizes"][0] * nm * C
    for i in range(1, a["n_blocks"] + 1):
        macs += 2 * C * C + (s - 1) * a["kernel_sizes"][i] * c8 * c8
    macs += a["n_blocks"] * C * M + M * A + A * M
    return 2 * macs


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:                                            # noqa: BLE001
        return f"unknown ({e})"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--modes", default="3xf16,f16,fp32,tf32")
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    g = np.random.default_rng(0)
    n = (g.uniform(1.0, 10.0, 64) * 16000).astype(int)
    wavs = [torch.from_numpy((0.1 * g.standard_normal(k)).astype(np.float32)) for k in n]
    x = torch.zeros(64, int(n.max()))
    for b, w in enumerate(wavs):
        x[b, : len(w)] = w
    x, lens = x.cuda(), torch.from_numpy(n).cuda()
    m = EO.seeded(0).cuda().eval()
    sd = m.state_dict()
    audio_s = float(n.sum()) / 16000
    frames = int((1 + n // 160).sum())
    encs = {mode: ECAPAEncoder(sd, mode) for mode in args.modes.split(",")}
    fpf = flops_per_frame(next(iter(encs.values())).arch)
    gw = [w.cuda() for w in wavs]

    def one_at_a_time():
        with torch.no_grad():
            for w in gw:
                m(EO.features(w)[None])

    def padded():
        with torch.no_grad():
            feats = [EO.features(w) for w in gw]
            T = max(f.shape[0] for f in feats)
            fb = torch.zeros(len(feats), T, 80, device="cuda")
            for b, f in enumerate(feats):
                fb[b, : f.shape[0]] = f
            m(fb)
    arms = {f"lib_{k}": (lambda e=e: e(x, lens)) for k, e in encs.items()}
    arms.update({"torch_fp32_one_at_a_time": one_at_a_time, "torch_fp32_padded_batch": padded})
    times = {k: [] for k in arms}
    for _ in range(2):                                                # alternate the arms
        for k, fn in arms.items():
            times[k].append(timed(fn, args.reps))
    res = {"card": card(), "batch": 64, "audio_seconds": round(audio_s, 2), "frames": frames,
           "gflop_per_frame_from_shapes": round(fpf / 1e9, 4), "arms": {}}
    for k, ts in times.items():
        t = min(ts)
        res["arms"][k] = {"seconds": round(t, 5), "audio_s_per_s": round(audio_s / t, 1), "tflops": round(fpf * frames / t / 1e12, 2)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
