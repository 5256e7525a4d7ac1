#!/usr/bin/env python
"""Multi-speaker FastSpeech2 (DESIGN.md section 25) on one H100, printed as one JSON line.  Writes nothing in the tree.

    python tools/bench_speakers.py [--steps 10] [--rounds 5]

Device events around `--steps` calls, median of `--rounds` windows; each pair of arms alternates window by window:
  synthesize_ms   `synthesize` at B = 64 on LJSpeech-shaped input (T = 100 phonemes, 3xf16), single-speaker model
                  against the same weights with a 109-row all-zero speaker table, so that both arms predict the same
                  durations and decode the same frames (the add is fused into the last encoder LayerNorm, so the
                  difference is expected inside the noise; a non-zero table changes the durations, hence the work)
  train_step_ms   a TF32 train step (forward + backward) at B = 16 and B = 64, T = 100, L = 800, without and with speakers
  backward_ms     fs2_speaker_add_backward alone at B = 64, T = 200, C = 256 for n in {109, 2456}
The card name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from statistics import median

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench_per_utterance import card  # noqa: E402


def paired(fns, steps, rounds):
    """Median ms per call of each fn, windows alternating between the fns."""
    for fn in fns:
        fn()
    torch.cuda.synchronize()
    out = [[] for _ in fns]
    for _ in range(rounds):
        for i, fn in enumerate(fns):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            out[i].append(e0.elapsed_time(e1) / steps)
    return [round(median(o), 3) for o in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_speakers needs a CUDA device")
    from fastspeech2_b200 import FeedForwardTransformer, _lib
    from fastspeech2_b200 import train as T
    from fastspeech2_b200.hparams import load_hp
    from fastspeech2_b200.synthetic import make_batch
    from fastspeech2_b200.weights import synthetic_state_dict

    sd = synthetic_state_dict(7)
    table = torch.randn(109, 256, generator=torch.Generator().manual_seed(1)) * 0.5

    def model(n, zero=False, **kw):
        hp = load_hp()
        hp["model"]["n_speakers"] = n
        m = FeedForwardTransformer(68, 80, hp, **kw)
        w = dict(sd)
        if n:
            w["speaker_embed.weight"] = torch.zeros(n, 256) if zero else table[:n]
        m.load_state_dict(w, strict=True)
        return m.cuda()

    res = {"workload": "LJSpeech-shaped synthetic, T = 100, L = 800"}
    # (a) synthesize, B = 64, 3xf16
    single, multi = model(0, precision="3xf16").eval(), model(109, zero=True, precision="3xf16").eval()
    bt = make_batch(64, 100, 800, seed=3, ilens=[100 - (b % 37) for b in range(64)])
    xs, il = bt["xs"].cuda(), bt["ilens"].cuda()
    spk = torch.randint(0, 109, (64,), generator=torch.Generator().manual_seed(2)).cuda()
    with torch.no_grad():
        a, b = paired([lambda: single.synthesize(xs, il), lambda: multi.synthesize(xs, il, speakers=spk)], args.steps, args.rounds)
        frames = int(single.synthesize(xs, il)[1].sum())
    res["synthesize_ms"] = {"B": 64, "precision": "3xf16", "frames": frames, "single": a, "speakers": b}
    del single, multi
    # (b) TF32 train step
    res["train_step_ms"] = {}
    for B in (16, 64):
        single, multi = model(0, train_precision="tf32").train(), model(109, train_precision="tf32").train()
        for m in (single, multi):
            m.dropout_masks = None
        tb = make_batch(B, 100, 800, seed=B)
        args_ = [tb[k].cuda() for k in ("xs", "ilens", "ys", "olens", "ds", "es", "ps")]
        sp = torch.randint(0, 109, (B,), generator=torch.Generator().manual_seed(B)).cuda()

        def step(m, **kw):
            loss, _ = m(*args_, **kw)
            loss.backward()
            for p in m.parameters():
                p.grad = None
        a, b = paired([lambda: step(single), lambda: step(multi, speakers=sp)], max(1, args.steps // 2), args.rounds)
        res["train_step_ms"][f"B={B}"] = {"single": a, "speakers": b}
        del single, multi
    # (c) fs2_speaker_add_backward alone
    lib = _lib.load()
    dy = torch.randn(64, 200, 256, device="cuda")
    nbytes = T.speaker_add_ws_bytes(64, 256)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    res["backward_ms"] = {}
    for n in (109, 2456):
        ids = torch.randint(0, n, (64,), generator=torch.Generator().manual_seed(n)).cuda()
        dt = torch.zeros(n, 256, device="cuda")
        st = _lib.stream_ptr(dy.device)
        fn = lambda: lib.fs2_speaker_add_backward(dy.data_ptr(), ids.data_ptr(), 64, 200, 256, n, dt.data_ptr(), ws.data_ptr(), nbytes, st)
        ms = paired([fn], 200, args.rounds)[0]
        res["backward_ms"][f"n={n}"] = {"ms": ms, "GB_per_s": round(64 * 200 * 256 * 4 / (ms * 1e-3) / 1e9, 1)}
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
