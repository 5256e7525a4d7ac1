#!/usr/bin/env python
"""Per-utterance batching (`model.synthesize`, `_forward(..., per_utterance=True)`) against the reference's batch
semantics on one H100, printed as one JSON line.  Writes nothing.

    python tools/bench_per_utterance.py [--precision 3xf16] [--steps 5] [--rounds 3]

Workloads:
  filelist64     inference on the 64 real LJSpeech phoneme sequences of tests/golden/filelist64.npz: ragged lengths,
                 where skipping the padding can gain;
  c2             inference on bench.py's c2 batch (B=64, T=100): the predicted lengths are ragged;
  c2_teacher_forced
                 bench.py's c2 teacher-forced step (every utterance T x L): no padding at all, so the mode must cost
                 nothing there;
  filelist64_controls
                 `synthesize` on filelist64 with explicit all-1.0 per-phoneme speed / pitch / energy against no controls:
                 the results are bit-identical, so the difference is the cost of the prosody-control path; plus a row
                 at speed 1.25 (25 % more frames), as valid frames/s.
Eager launches, one host read per inference call; the two semantics run in alternating windows of `--steps` calls,
and each reports the median window of `--rounds`.  The card name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def padding_share(olens, Lmax: int, tile: int = 128) -> dict:
    """Fraction of the MMA rows of a row-wise GEMM that fall on padding, from shapes: the [B, Lmax] rectangle, against
    per-utterance 128-row tiles with the tiles wholly past each length skipped."""
    valid = sum(olens)
    tiled = sum(-(-n // tile) * tile for n in olens)
    return {"rectangle": 1.0 - valid / (len(olens) * Lmax), "per_utterance_tiles": 1.0 - valid / tiled}


def alternate(fns: dict, steps: int, rounds: int) -> dict:
    """name -> per-call ms of each of `rounds` alternating windows of `steps` calls (after one warm-up call each)."""
    ms = {name: [] for name in fns}
    with torch.no_grad():
        for fn in fns.values():
            fn()
        for _ in range(rounds):
            for name, fn in fns.items():
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(steps):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                ms[name].append(e0.elapsed_time(e1) / steps)
    return ms


def median(v):
    return sorted(v)[len(v) // 2]


def inference_semantics(model, xs, ilens, steps: int, rounds: int) -> dict:
    def ref():
        return model._forward(xs, ilens, is_inference=True, _one_hot=False)

    def per_utt():
        return model.synthesize(xs, ilens)

    with torch.no_grad():
        r, p = ref(), per_utt()
        shapes = {"reference": ([int(v) for v in r[2].sum(1).tolist()], int(r[1].shape[1])),
                  "per_utterance": ([int(v) for v in p[1].tolist()], int(p[0].shape[1]))}
    ms = alternate({"reference": ref, "per_utterance": per_utt}, steps, rounds)
    out = {}
    for name, (olens, Lmax) in shapes.items():
        t = median(ms[name])
        out[name] = {"value": sum(olens) / (t * 1e-3), "unit": "valid frames/s", "ms_per_step": t, "ms_windows": ms[name],
                     "Lmax": Lmax, "valid_frames": sum(olens), "padding_rows_share": padding_share(olens, Lmax)}
    out["speedup"] = out["reference"]["ms_per_step"] / out["per_utterance"]["ms_per_step"]
    out["note"] = (f"B={int(xs.shape[0])}; reference semantics: the decoder runs every row of the [B,Lmax] rectangle, "
                   "unmasked (batch mates can change an utterance's durations, so its frame count may differ); "
                   "per-utterance: model.synthesize, each utterance bit-identical to its B=1 inference")
    return out


def teacher_forced_semantics(model, batch, steps: int, rounds: int) -> dict:
    args = [batch[k] for k in ("xs", "ilens", "olens", "ds", "es", "ps")]
    ms = alternate({"reference": lambda: model._forward(*args, is_inference=False),
                    "per_utterance": lambda: model._forward(*args, is_inference=False, per_utterance=True)}, steps, rounds)
    med = {k: median(v) for k, v in ms.items()}
    return {"ms_per_step": med, "ms_windows": ms, "per_utterance_over_reference": med["per_utterance"] / med["reference"]}


def controls_cost(model, xs, ilens, steps: int, rounds: int) -> dict:
    ones = torch.ones(xs.shape, device=xs.device)
    fns = {"none": lambda: model.synthesize(xs, ilens),
           "neutral": lambda: model.synthesize(xs, ilens, speed=ones, pitch=ones, energy=ones),
           "speed_1.25": lambda: model.synthesize(xs, ilens, speed=1.25 * ones, pitch=ones, energy=ones)}
    with torch.no_grad():
        outs = {name: fn() for name, fn in fns.items()}
    assert all(torch.equal(a, b) for a, b in zip(outs["none"], outs["neutral"])), "all-1.0 controls changed the result"
    ms = alternate(fns, steps, rounds)
    out = {}
    for name, (_, olens, _) in outs.items():
        t, frames = median(ms[name]), int(olens.sum())
        out[name] = {"value": frames / (t * 1e-3), "unit": "valid frames/s", "ms_per_step": t, "ms_windows": ms[name],
                     "valid_frames": frames}
    out["neutral_over_none"] = out["neutral"]["ms_per_step"] / out["none"]["ms_per_step"]
    return out


def card() -> dict:
    info = {"name": torch.cuda.get_device_name()}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=20)
        info["power_limit"] = r.stdout.strip() or None
    except Exception:
        info["power_limit"] = None
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default=os.environ.get("FS2_PRECISION", "3xf16"), choices=["fp32", "tf32", "3xtf32", "3xf16", "f16"])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.hparams import load_hp
    from fastspeech2_b200.synthetic import make_batch

    dev = torch.device("cuda", torch.cuda.current_device())
    model = FeedForwardTransformer(68, 80, load_hp(), precision=args.precision)
    model.load_state_dict(synthetic_state_dict(0), strict=True)        # bench.py's checkpoint and c2 batch
    model = model.to(dev).eval()
    c2 = {k: v.to(dev) for k, v in make_batch(64, 100, 800, seed=1234).items()}
    fl = np.load(os.path.join(ROOT, "tests", "golden", "filelist64.npz"))
    line = {
        "metric": "per-utterance vs reference-semantics batched synthesis; cost of prosody controls", "precision": args.precision, "card": card(),
        "filelist64": inference_semantics(model, torch.from_numpy(fl["xs"]).to(dev), torch.from_numpy(fl["ilens"]).to(dev),
                                          args.steps, args.rounds),
        "c2": inference_semantics(model, c2["xs"], c2["ilens"], args.steps, args.rounds),
        "c2_teacher_forced": teacher_forced_semantics(model, c2, args.steps, args.rounds),
        "filelist64_controls": controls_cost(model, torch.from_numpy(fl["xs"]).to(dev), torch.from_numpy(fl["ilens"]).to(dev),
                                             args.steps, args.rounds),
        "timing": f"eager launches, alternating windows of {args.steps} calls, median of {args.rounds} windows per semantics",
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
