#!/usr/bin/env python
"""Phonemes to audio, eager against CUDA-graph replay (`graphed_synthesize`), printed as one JSON line.  Writes nothing.

    python tools/bench_graphed_synthesis.py [--steps 10] [--rounds 7]

Model: random-init weights (synthetic_state_dict(0), only the lengths matter for time) in 3xf16; vocoders HiFi-GAN V3
and MelGAN with random-init weights in 3xf16.  For each vocoder:
  eager               model.synthesize(xs, ilens) then vocoder(mels, olens): two host reads per request;
  graph_{1.0,1.5,2.0}x one replay of a graph captured at capacity = that multiple of the batch's Lmax (validate=True:
                      one status-word copy per replay).
Workloads:
  b1      B = 1, the 50-phoneme utterance of make_batch(1, 50, 400, seed=7) that bench.py's latency figure uses; host
          wall-clock per request, each request ending in a device synchronize;
  b8      the first 8 utterances of tests/golden/filelist64.npz; device time per batch (CUDA events);
  b64     all 64 of them; device time per batch.
The variants of a workload run in alternating windows of `--steps` requests, median of `--rounds` windows.  The card's
name and power limit are read in the same run.
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

from bench_per_utterance import alternate, card, median  # noqa: E402

CAPACITIES = (1.0, 1.5, 2.0)


def host_alternate(fns: dict, steps: int, rounds: int) -> dict:
    """name -> per-request host ms of each of `rounds` alternating windows of `steps` requests, each ending in a
    synchronize (after one warm-up request each)."""
    ms = {name: [] for name in fns}
    with torch.no_grad():
        for fn in fns.values():
            fn()
            torch.cuda.synchronize()
        for _ in range(rounds):
            for name, fn in fns.items():
                t0 = time.perf_counter()
                for _ in range(steps):
                    fn()
                    torch.cuda.synchronize()
                ms[name].append((time.perf_counter() - t0) * 1e3 / steps)
    return ms


def workload(model, voc, xs, ilens, host: bool, steps: int, rounds: int) -> dict:
    with torch.no_grad():
        mels, olens, _ = model.synthesize(xs, ilens)
    lmax = int(mels.shape[1])
    B, T = xs.shape

    def eager():
        m, o, _ = model.synthesize(xs, ilens)
        return voc(m, o)

    fns = {"eager": eager}
    graphs = {}
    for f in CAPACITIES:
        cap = int(round(f * lmax))
        g = graphs[f] = model.graphed_synthesize(B, T, cap, vocoder=voc)
        fns[f"graph_{f:.1f}x"] = (lambda g=g: g(xs, ilens))
    # the graph's slots against the eager path on this batch, bit for bit, before any timing
    with torch.no_grad():
        audio_e, alens_e = eager()
        for g in graphs.values():
            _, o, _, audio, alens = g(xs, ilens)
            assert torch.equal(o, olens) and torch.equal(alens, alens_e)
            for b in range(B):
                n = int(alens[b])
                assert torch.equal(audio[b, :n], audio_e[b, :n]), b
    ms = (host_alternate if host else alternate)(fns, steps, rounds)
    row = {"B": B, "Tmax": T, "Lmax": lmax, "frames": int(olens.sum()), "timer": "host_wallclock" if host else "cuda_events"}
    for name, v in ms.items():
        row[f"{name}_ms"] = round(median(v), 3)
        row[f"{name}_ms_spread"] = [round(min(v), 3), round(max(v), 3)]
    for f in CAPACITIES:
        row[f"graph_{f:.1f}x_capacity"] = graphs[f].capacity
        row[f"speedup_{f:.1f}x"] = round(row["eager_ms"] / row[f"graph_{f:.1f}x_ms"], 3)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_graphed_synthesis needs a CUDA device")
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.hifigan import HiFiGANVocoder
    from fastspeech2_b200.hparams import load_hp
    from fastspeech2_b200.melgan import MelGANVocoder
    from fastspeech2_b200.synthetic import make_batch

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model = FeedForwardTransformer(68, 80, load_hp(), precision="3xf16")
    model.load_state_dict(synthetic_state_dict(0), strict=True)
    model = model.to(dev).eval()
    torch.manual_seed(0)
    vocoders = {"hifigan_v3": HiFiGANVocoder("v3", math_mode="3xf16").to(dev), "melgan": MelGANVocoder(math_mode="3xf16").to(dev)}
    fl = np.load(os.path.join(ROOT, "tests", "golden", "filelist64.npz"))
    x1 = make_batch(1, 50, 400, seed=7)["xs"].to(dev)
    loads = {
        "b1": (x1, torch.tensor([50], device=dev), True),
        "b8": (torch.from_numpy(fl["xs"][:8]).to(dev), torch.from_numpy(fl["ilens"][:8]).to(dev), False),
        "b64": (torch.from_numpy(fl["xs"]).to(dev), torch.from_numpy(fl["ilens"]).to(dev), False),
    }
    out = {"card": card(), "precision": "3xf16", "steps": args.steps, "rounds": args.rounds}
    for vname, voc in vocoders.items():
        for lname, (xs, il, host) in loads.items():
            xs = xs[:, : int(il.max())].contiguous()
            out[f"{vname}_{lname}"] = workload(model, voc, xs, il, host, args.steps, args.rounds)
            print(vname, lname, json.dumps(out[f"{vname}_{lname}"]), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
