#!/usr/bin/env python
"""One full train step (forward, backward, clip_grad_norm_, Adam) in train_precision fp32 and tf32 on one H100, printed
as one JSON line.  Writes nothing.

    python tools/bench_train.py [--rounds 3] [--window-s 1.0] [--workloads filelist16,c2]

Workloads (random-init weights, synthetic_state_dict(0)):
  filelist16  the first 16 utterances of tests/golden/filelist64.npz (the reference's batch size) with their MFA
              durations; energy, pitch and target mels drawn from a seeded generator;
  c2          bench.py's shapes: B = 64, T = 100, L = 800 (make_batch seed 1234).
Each mode has its own model and Adam optimizer (lr 1e-4); the two steps alternate in windows of about --window-s seconds
(CUDA events, synchronised), and each mode reports the median of --rounds windows.  Before timing, both modes take one
step from the same weights on the timed batch and their losses and gradient norms are compared.  A separate
torch.profiler pass per mode gives device time per class: ConvFn forward (tap GEMM + weight packing launched in the
forward phase), dgrad (the same, launched in the backward phase), wgrad (weight-gradient kernels, their tf32 transposes
and split-K reduce, and the bias column sums), attention (the batched score / context products and the softmax
kernels), and the rest.  The wgrad rate is 2 B L N K taps summed over the step's ConvFn calls, over the wgrad main
kernel's device time, against the data sheet's 495 TFLOP/s dense TF32.  The card name, power limit and max SM clock are
read in the same run.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

TF32_TFLOPS = 495.0
KEYS = ("xs", "ilens", "ys", "olens", "ds", "es", "ps")


def card() -> dict:
    info = {"name": torch.cuda.get_device_name()}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=20)
        parts = [p.strip() for p in r.stdout.strip().split(",")]
        info["power_limit"], info["max_sm_clock"] = (parts + [None, None])[:2]
    except Exception:
        info["power_limit"] = info["max_sm_clock"] = None
    return info


def workload(name: str, dev) -> dict:
    from fastspeech2_b200.synthetic import make_batch
    if name == "c2":
        return {k: v.to(dev) for k, v in make_batch(64, 100, 800, seed=1234).items()}
    fl = np.load(os.path.join(ROOT, "tests", "golden", "filelist64.npz"))
    ilens = torch.from_numpy(fl["ilens"][:16])
    T = int(ilens.max())
    ds = torch.from_numpy(fl["ds"][:16, :T])
    olens = ds.sum(1)
    L = int(olens.max())
    g = torch.Generator().manual_seed(16)
    return {"xs": torch.from_numpy(fl["xs"][:16, :T]).to(dev), "ilens": ilens.to(dev), "ds": ds.to(dev), "olens": olens.to(dev),
            "es": (torch.rand(16, L, generator=g) * 60).to(dev), "ps": (80 + torch.rand(16, L, generator=g) * 300).to(dev),
            "ys": torch.randn(16, L, 80, generator=g).to(dev)}


def make(mode: str, dev):
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.hparams import load_hp
    m = FeedForwardTransformer(68, 80, load_hp(), train_precision=mode)
    m.load_state_dict(synthetic_state_dict(0), strict=True)
    m = m.to(dev).train()
    return m, torch.optim.Adam(m.parameters(), lr=1e-4)


def step(m, opt, batch):
    loss, _ = m(*[batch[k] for k in KEYS])
    loss.backward()
    gn = torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0)
    opt.step()
    opt.zero_grad(set_to_none=True)
    return loss, gn


def compare(models, batch) -> dict:
    """One forward + backward per mode from the same weights: loss, global gradient norm, worst per-parameter difference."""
    out, grads = {}, {}
    for mode, (m, _) in models.items():
        loss, _ = m(*[batch[k] for k in KEYS])
        loss.backward()
        grads[mode] = {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}
        out[mode] = {"loss": float(loss.detach()), "grad_norm": float(torch.linalg.vector_norm(torch.stack([g.norm() for g in grads[mode].values()])))}
        m.zero_grad(set_to_none=True)
    worst = max(((float((grads["tf32"][n] - g).norm() / (g.norm() + 1e-30)), n) for n, g in grads["fp32"].items()))
    out["loss_rel_diff"] = abs(out["tf32"]["loss"] - out["fp32"]["loss"]) / abs(out["fp32"]["loss"])
    out["grad_norm_rel_diff"] = abs(out["tf32"]["grad_norm"] - out["fp32"]["grad_norm"]) / out["fp32"]["grad_norm"]
    out["worst_param_grad_rel_diff"] = {"param": worst[1], "value": worst[0]}
    return out


def timed(models, batch, rounds: int, window_s: float) -> dict:
    for m, opt in models.values():         # warm-up: every shape of the window
        step(m, opt, batch)
    torch.cuda.synchronize()
    per = {}
    for mode, (m, opt) in models.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); step(m, opt, batch); e1.record(); torch.cuda.synchronize()
        per[mode] = e0.elapsed_time(e1)
    n = max(3, math.ceil(window_s * 1e3 / min(per.values())))
    ms = {mode: [] for mode in models}
    for _ in range(rounds):
        for mode, (m, opt) in models.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                step(m, opt, batch)
            e1.record()
            torch.cuda.synchronize()
            ms[mode].append(e0.elapsed_time(e1) / n)
    med = {mode: sorted(v)[len(v) // 2] for mode, v in ms.items()}
    return {"steps_per_window": n, "ms_per_step": med, "ms_windows": ms, "tf32_speedup": med["fp32"] / med["tf32"]}


def classify(name: str, phase: str) -> str:
    if any(s in name for s in ("wgrad", "transpose_tf32", "colsum")):
        return "wgrad"
    if "tap_gemm" in name or "pack_conv_weight" in name or "pack_dgrad_weight" in name:
        return "dgrad" if phase == "bwd" else "forward"
    if any(s in name for s in ("bgemm", "attn_softmax")):
        return "attention"
    return "rest"


def profiled(m, opt, batch) -> dict:
    from torch.profiler import ProfilerActivity, profile, record_function
    from fastspeech2_b200 import train as T
    flops = []
    apply = T.ConvFn.apply

    def recording(x, w, *rest):
        B, L, K = x.shape
        flops.append(2.0 * B * L * w.shape[0] * K * (w.shape[2] if w.dim() == 3 else 1))
        return apply(x, w, *rest)

    step(m, opt, batch)
    torch.cuda.synchronize()
    T.ConvFn.apply = recording
    try:
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            with record_function("fwd"):
                loss, _ = m(*[batch[k] for k in KEYS])
                torch.cuda.synchronize()
            with record_function("bwd"):
                loss.backward()
                torch.cuda.synchronize()
            with record_function("opt"):
                torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0)
                opt.step()
                opt.zero_grad(set_to_none=True)
                torch.cuda.synchronize()
    finally:
        del T.ConvFn.apply
    with tempfile.TemporaryDirectory() as tmp:        # the trace's kernel and annotation timestamps share one timeline
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        trace = json.load(open(path))["traceEvents"]
    starts = {e["name"]: e["ts"] for e in trace if e.get("cat") == "user_annotation" and e.get("name") in ("fwd", "bwd", "opt")}
    us = {c: 0.0 for c in ("forward", "dgrad", "wgrad", "attention", "rest")}
    wgrad_main = 0.0
    for e in trace:
        if e.get("cat") != "kernel":
            continue
        phase = "fwd" if e["ts"] < starts["bwd"] else "bwd" if e["ts"] < starts["opt"] else "opt"
        us[classify(e["name"], phase)] += e["dur"]
        if "wgrad_tc_kernel" in e["name"] or "wgrad_kernel" in e["name"]:
            wgrad_main += e["dur"]
    wg_flop = sum(flops)    # the weight gradient costs what the forward costs: 2 B L N K taps per ConvFn
    total = sum(us.values())
    return {"device_ms": {c: v / 1e3 for c, v in us.items()}, "device_ms_total": total / 1e3,
            "share": {c: v / total for c, v in us.items()},
            "wgrad_gflop": wg_flop / 1e9, "wgrad_main_kernel_ms": wgrad_main / 1e3,
            "wgrad_main_kernel_tflops": wg_flop / (wgrad_main * 1e-6) / 1e12 if wgrad_main else None,
            "wgrad_class_tflops": wg_flop / (us["wgrad"] * 1e-6) / 1e12 if us["wgrad"] else None,
            "wgrad_main_kernel_share_of_tf32_bound": (wg_flop / (wgrad_main * 1e-6) / 1e12) / TF32_TFLOPS if wgrad_main else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window-s", type=float, default=1.0)
    ap.add_argument("--workloads", default="filelist16,c2")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    line = {"metric": "train step (forward, backward, clip_grad_norm_, Adam), train_precision fp32 vs tf32", "card": card(),
            "tf32_bound_tflops": TF32_TFLOPS}
    for name in args.workloads.split(","):
        batch = workload(name, dev)
        models = {mode: make(mode, dev) for mode in ("fp32", "tf32")}
        row = {"B": int(batch["xs"].shape[0]), "T": int(batch["xs"].shape[1]), "L": int(batch["olens"].max()),
               "valid_frames": int(batch["olens"].sum())}
        row["numerics"] = compare(models, batch)
        row["timing"] = timed(models, batch, args.rounds, args.window_s)
        row["profile"] = {mode: profiled(m, opt, batch) for mode, (m, opt) in models.items()}
        line[name] = row
        del models
        torch.cuda.empty_cache()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
