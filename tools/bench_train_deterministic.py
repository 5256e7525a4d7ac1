#!/usr/bin/env python
"""What the deterministic train mode costs (DESIGN.md §26): one full train step (forward, backward, NoamAdam.clip_and_step)
with train_deterministic off and on, in fp32, tf32 and tf32 + flash, printed as one JSON line.  Writes nothing.

    python tools/bench_train_deterministic.py [--rounds 3] [--window-s 1.0] [--workloads filelist16,c2] [--modes fp32,tf32,flash]

Workloads are tools/bench_train.py's (filelist16: the reference's batch of 16 utterances; c2: B = 64, T = 100, L = 800).
For each (workload, mode) a default and a deterministic model start from the same weights; after a warm-up step each,
the two arms alternate in windows of about --window-s seconds timed with CUDA events, and each arm reports the median of
--rounds windows.  A separate torch.profiler pass per arm gives the device time of every site the mode replaces (the
ordered kernels against the atomic kernels they stand in for).  The extra workspace of the c2 step is the largest
ordered workspace any one call of that step takes.  The card name, power limit and max SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench_train import KEYS, card, workload  # noqa: E402

MODES = {"fp32": ("fp32", "materialized"), "tf32": ("tf32", "materialized"), "flash": ("tf32", "flash")}
# ordered kernel -> the site it belongs to (its default kernel carries the same site name)
SITES = (("colsum", "bias column sums"), ("wgrad_kernel", "fp32 weight gradient"), ("wgrad_reduce", "fp32 weight gradient"),
         ("layernorm_backward", "LayerNorm backward"), ("bn_", "BatchNorm"), ("embed_backward", "embedding scatter"),
         ("onehot_linear_backward", "one-hot scatter"), ("scatter_", "id scatter (sort and sums)"), ("rowdot_backward", "predictor heads"),
         ("loss_", "loss sums"), ("ordered_sum_f64", "double sums (BatchNorm, loss)"))


def make(prec, att, det, dev):
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200 import optim as O
    from fastspeech2_b200.hparams import load_hp
    m = FeedForwardTransformer(68, 80, load_hp(), train_precision=prec, train_attention=att, train_deterministic=det)
    m.load_state_dict(synthetic_state_dict(0), strict=True)
    m = m.to(dev).train()
    return m, O.get_std_opt(m, 384, 4000, 1.0)


def step(m, opt, batch):
    loss, _ = m(*[batch[k] for k in KEYS])
    loss.backward()
    opt.clip_and_step(1.0)
    opt.zero_grad()
    return loss


def timed(arms, batch, rounds, window_s):
    for m, opt in arms.values():
        step(m, opt, batch)
    torch.cuda.synchronize()
    one = {}
    for k, (m, opt) in arms.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); step(m, opt, batch); e1.record(); torch.cuda.synchronize()
        one[k] = e0.elapsed_time(e1)
    n = max(3, math.ceil(window_s * 1e3 / min(one.values())))
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, (m, opt) in arms.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                step(m, opt, batch)
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / n)
    med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
    return {"steps_per_window": n, "ms_per_step": med, "ms_windows": ms, "slowdown": med["deterministic"] / med["default"] - 1.0}


def site_of(name):
    for key, site in SITES:
        if key in name:
            return site
    return None


def profiled(m, opt, batch):
    from torch.profiler import ProfilerActivity, profile
    step(m, opt, batch)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(m, opt, batch)
        torch.cuda.synchronize()
    per, total = {}, 0.0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        total += us
        s = site_of(e.name)
        if s:
            per[s] = per.get(s, 0.0) + us / 1e3
    return {"device_ms_total": total / 1e3, "site_ms": {k: round(v, 4) for k, v in sorted(per.items())}}


def c2_workspace_bytes():
    """the largest ordered workspace a c2 step asks for (the per-call size queries at the step's shapes)"""
    from fastspeech2_b200._kernel_module import query_bytes
    B, T, L = 64, 100, 800
    sizes = {
        "layernorm_backward (decoder rows)": query_bytes("fs2_layernorm_backward_det_ws_bytes", B * L, 384),
        "onehot_linear_backward (256 bins)": query_bytes("fs2_onehot_linear_backward_det_ws_bytes", B * L, 384, 256),
        "embed_backward (encoder table)": query_bytes("fs2_embed_backward_det_ws_bytes", B, T, 384, 68),
        "embed_backward (decoder positions)": query_bytes("fs2_embed_backward_det_ws_bytes", B, L, 384, 0),
        "rowdot_backward (frame heads)": query_bytes("fs2_rowdot_backward_det_ws_bytes", B * L, 256),
        "conv_wgrad fp32 (conv-FFN w_1)": query_bytes("fs2_conv_wgrad_det_ws_bytes", B, L, 1024, 384, 9),
        "batchnorm (Postnet)": query_bytes("fs2_batchnorm_backward_det_ws_bytes", B * L, 256),
        "masked_losses": query_bytes("fs2_masked_losses_det_ws_bytes", B, T, L, 80),
    }
    return {"max_bytes": max(sizes.values()), "per_call_bytes": sizes}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window-s", type=float, default=1.0)
    ap.add_argument("--workloads", default="filelist16,c2")
    ap.add_argument("--modes", default="fp32,tf32,flash")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda")
    line = {"bench": "train_deterministic", "card": card(), "results": {}}
    for wl in args.workloads.split(","):
        batch = workload(wl, dev)
        for mode in args.modes.split(","):
            prec, att = MODES[mode]
            arms = {"default": make(prec, att, False, dev), "deterministic": make(prec, att, True, dev)}
            r = timed(arms, batch, args.rounds, args.window_s)
            r["profile"] = {k: profiled(m, opt, batch) for k, (m, opt) in arms.items()}
            line["results"][f"{wl}/{mode}"] = r
            del arms
            torch.cuda.empty_cache()
    line["c2_extra_workspace"] = c2_workspace_bytes()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
