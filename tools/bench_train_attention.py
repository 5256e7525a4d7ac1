#!/usr/bin/env python
"""The TF32 train step with materialized attention against the fused flash attention (train_attention="flash") on one
H100, printed as one JSON line.  Writes nothing.

    python tools/bench_train_attention.py [--rounds 3] [--window-s 1.0] [--workloads filelist16,c2,long]

Workloads (random-init weights, synthetic_state_dict(0)): filelist16 and c2 as in tools/bench_train.py, and
  long  B = 8, T = 400, L = 3200 (make_batch seed 77): the materialized path saves 9 bytes per score element, about
        0.7 GB per decoder layer here.
Both modes train in tf32 with their own model and Adam optimizer; steps alternate in windows of about --window-s seconds
(CUDA events), median of --rounds windows.  Before timing, both take one Philox-seeded step from the same weights and
their losses and gradient norms are compared.  Peak torch.cuda.max_memory_allocated over one step, per mode.  A
torch.profiler pass per mode gives device time per class as in tools/bench_train.py; the attention class counts the
batched products and softmax kernels (materialized) or the fused kernels, their rounding prep pass and D (flash).
The card name, power limit and max SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import torch  # noqa: E402

import bench_train as BT  # noqa: E402

MODES = ("materialized", "flash")
_base_classify = BT.classify


def workload(name: str, dev) -> dict:
    if name == "long":
        from fastspeech2_b200.synthetic import make_batch
        return {k: v.to(dev) for k, v in make_batch(8, 400, 3200, seed=77).items()}
    return BT.workload(name, dev)


def make(mode: str, dev):
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.hparams import load_hp
    m = FeedForwardTransformer(68, 80, load_hp(), train_precision="tf32", train_attention=mode)
    m.load_state_dict(synthetic_state_dict(0), strict=True)
    m = m.to(dev).train()
    return m, torch.optim.Adam(m.parameters(), lr=1e-4)


def compare(models, batch) -> dict:
    from fastspeech2_b200 import train as T
    out = {}
    for mode, (m, _) in models.items():
        m.dropout_masks = T.MaskSource(seed=4321)
        loss, _ = m(*[batch[k] for k in BT.KEYS])
        loss.backward()
        gn = torch.linalg.vector_norm(torch.stack([p.grad.norm() for p in m.parameters() if p.grad is not None]))
        out[mode] = {"loss": float(loss.detach()), "grad_norm": float(gn), "mask_offset": m.dropout_masks.offset}
        m.dropout_masks = None
        m.zero_grad(set_to_none=True)
    a, b = out["materialized"], out["flash"]
    out["loss_rel_diff"] = abs(b["loss"] - a["loss"]) / abs(a["loss"])
    out["grad_norm_rel_diff"] = abs(b["grad_norm"] - a["grad_norm"]) / a["grad_norm"]
    return out


def timed(models, batch, rounds: int, window_s: float) -> dict:
    for m, opt in models.values():
        BT.step(m, opt, batch)
    torch.cuda.synchronize()
    per = {}
    for mode, (m, opt) in models.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); BT.step(m, opt, batch); e1.record(); torch.cuda.synchronize()
        per[mode] = e0.elapsed_time(e1)
    n = max(3, math.ceil(window_s * 1e3 / min(per.values())))
    ms = {mode: [] for mode in models}
    for _ in range(rounds):
        for mode, (m, opt) in models.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                BT.step(m, opt, batch)
            e1.record()
            torch.cuda.synchronize()
            ms[mode].append(e0.elapsed_time(e1) / n)
    med = {mode: sorted(v)[len(v) // 2] for mode, v in ms.items()}
    return {"steps_per_window": n, "ms_per_step": med, "ms_windows": ms, "flash_speedup": med["materialized"] / med["flash"]}


def peak_memory(m, opt, batch) -> dict:
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    BT.step(m, opt, batch)
    torch.cuda.synchronize()
    return {"peak_gb": torch.cuda.max_memory_allocated() / 1e9, "rise_gb": (torch.cuda.max_memory_allocated() - base) / 1e9}


def classify(name: str, phase: str) -> str:
    if "attn_" in name and "attn_softmax" not in name:          # the fused kernels: attn_fwd / dkdv / dq / delta / round
        return "attention"
    return _base_classify(name, phase)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window-s", type=float, default=1.0)
    ap.add_argument("--workloads", default="filelist16,c2,long")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    BT.classify = classify
    line = {"metric": "tf32 train step (forward, backward, clip_grad_norm_, Adam), materialized vs flash attention", "card": BT.card()}
    for name in args.workloads.split(","):
        batch = workload(name, dev)
        row = {"B": int(batch["xs"].shape[0]), "T": int(batch["xs"].shape[1]), "L": int(batch["olens"].max()),
               "valid_frames": int(batch["olens"].sum())}
        models = {mode: make(mode, dev) for mode in MODES}
        row["numerics"] = compare(models, batch)
        row["timing"] = timed(models, batch, args.rounds, args.window_s)
        row["profile"] = {}
        for mode, (m, opt) in models.items():
            p = BT.profiled(m, opt, batch)
            row["profile"][mode] = {"device_ms": p["device_ms"], "device_ms_total": p["device_ms_total"], "share": p["share"]}
        del models
        torch.cuda.empty_cache()
        row["memory"] = {}
        for mode in MODES:                    # one mode's model at a time, so each peak is its own
            m, opt = make(mode, dev)
            BT.step(m, opt, batch)
            row["memory"][mode] = peak_memory(m, opt, batch)
            del m, opt
            torch.cuda.empty_cache()
        line[name] = row
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
