#!/usr/bin/env python
"""Objective evaluation on one H100 (`mcd_dtw`, `path_prosody`), printed as one JSON line.  Writes nothing in the tree.

    python tools/bench_evaluate.py [--steps 5] [--rounds 3] [--oracle-pairs 2] [--profile]

Workload: B = 64 LJSpeech-shaped pairs, seeded: reference lengths U[150, 870] frames, synthesized / reference length
ratio U[0.8, 1.25], 80 smooth random-walk log-mels per frame, n_cep = 24, F0 contours with about 30 % unvoiced frames.
  mcd             mcd_dtw without a path (cepstra and the wavefront sweep)
  mcd_path        mcd_dtw with the path (direction bytes and the backtrack)
  mcd_prosody     mcd_dtw with the path, then path_prosody: what the evaluate command runs per batch
each as device events around `--steps` calls, median of `--rounds` windows: ms per batch, pairs/s, and DTW cells/s
(sum of Lx * Ly over the time).  `--profile` adds per-kernel device time from torch.profiler, in a separate run.
  oracle          the float64 numpy restatement (oracle/eval_oracle.py) on the first `--oracle-pairs` pairs on the CPU,
                  for context, and whether the GPU's cost, path and MCD match it bit for bit there.
The card name and power limit are read in the same run.
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

from bench_per_utterance import card, median  # noqa: E402

B, M, N_CEP = 64, 80, 24


def workload(seed=0):
    rng = np.random.default_rng(seed)
    ly = rng.integers(150, 871, B)
    lx = np.maximum(1, np.round(ly * rng.uniform(0.8, 1.25, B))).astype(int)

    def mel(n):
        walk = np.cumsum(rng.standard_normal((n, M)) * 0.3, axis=0)
        return np.clip(-5 + walk - np.linspace(0, 4, M)[None] + rng.standard_normal((n, M)) * 0.2, -11.5, 2).astype(np.float32)

    def f0(n):
        return np.where(rng.random(n) < 0.3, 0.0, 120 * np.exp(0.2 * np.cumsum(rng.standard_normal(n)) / np.sqrt(n)))
    xs, ys = [mel(n) for n in lx], [mel(n) for n in ly]
    fxs, fys = [f0(n) for n in lx], [f0(n) for n in ly]
    exs, eys = [rng.uniform(0, 20, n).astype(np.float32) for n in lx], [rng.uniform(0, 20, n).astype(np.float32) for n in ly]
    return lx, ly, xs, ys, fxs, fys, exs, eys


def pad(arrs, dtype):
    n = [a.shape[0] for a in arrs]
    out = torch.zeros((len(arrs), max(n)) + tuple(arrs[0].shape[1:]), dtype=dtype)
    for b, a in enumerate(arrs):
        out[b, : n[b]] = torch.as_tensor(a, dtype=dtype)
    return out.cuda(), torch.tensor(n).cuda()


def timed(fn, steps, rounds):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / steps)
    return median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--oracle-pairs", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_evaluate needs a CUDA device")
    from fastspeech2_b200 import evaluate as EV
    from oracle import eval_oracle as E

    lx, ly, xs, ys, fxs, fys, exs, eys = workload()
    x, xl = pad(xs, torch.float32)
    y, yl = pad(ys, torch.float32)
    fx, fxl = pad(fxs, torch.float64)
    fy, fyl = pad(fys, torch.float64)
    ex, _ = pad(exs, torch.float32)
    ey, _ = pad(eys, torch.float32)
    cells = float(np.sum(lx.astype(np.int64) * ly))

    def mcd():
        return EV.mcd_dtw(x, xl, y, yl, n_cep=N_CEP)

    def mcd_path():
        return EV.mcd_dtw(x, xl, y, yl, n_cep=N_CEP, return_path=True)

    def mcd_prosody():
        r = mcd_path()
        return EV.path_prosody(r[3], r[2], fx, fxl, fy, fyl, ex, ey)

    out = {"metric": "objective evaluation, B = 64 LJSpeech-shaped pairs", "card": card(), "B": B, "n_mels": M, "n_cep": N_CEP,
           "Lx_max": int(lx.max()), "Ly_max": int(ly.max()), "cells": int(cells),
           "workspace_bytes": {"mcd": EV.workspace_bytes(B, int(lx.max()), int(ly.max()), M, N_CEP, False),
                               "mcd_path": EV.workspace_bytes(B, int(lx.max()), int(ly.max()), M, N_CEP, True)}}
    for name, fn in (("mcd", mcd), ("mcd_path", mcd_path), ("mcd_prosody", mcd_prosody)):
        ms = timed(fn, args.steps, args.rounds)
        out[name] = {"ms_per_batch": round(ms, 3), "pairs_per_s": round(B / ms * 1e3, 1), "cells_per_s": float(f"{cells / ms * 1e3:.4g}")}

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        mcd_prosody()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                mcd_prosody()
            torch.cuda.synchronize()
        per = {}
        for e in prof.events():
            if e.device_type.name == "CUDA" and "eval_" in e.name:
                k = e.name.split("eval_")[1].split("_kernel")[0]
                per[k] = per.get(k, 0.0) + e.device_time / 1e3 / args.steps
        out["kernel_ms"] = {k: round(v, 3) for k, v in sorted(per.items())}

    n = args.oracle_pairs
    mcd_g, cost_g, plen_g, path_g = (t.cpu().numpy() for t in mcd_path())
    D = EV.dct_basis(M, N_CEP)
    t0 = time.perf_counter()
    want = [E.evaluate_pair(xs[b], ys[b], D) for b in range(n)]
    dt = time.perf_counter() - t0
    match = all(cost_g[b] == w["cost"] and mcd_g[b] == w["mcd"] and plen_g[b] == w["plen"]
                and np.array_equal(path_g[b, : w["plen"]], w["path"]) for b, w in enumerate(want))
    ocells = float(np.sum(lx[:n].astype(np.int64) * ly[:n]))
    out["oracle"] = {"pairs": n, "s_per_pair": round(dt / n, 3), "cells_per_s": float(f"{ocells / dt:.4g}"), "bit_identical": bool(match)}
    out["speedup_vs_oracle"] = round((dt / n) / (out["mcd_prosody"]["ms_per_batch"] / 1e3 / B), 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
