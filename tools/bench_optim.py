#!/usr/bin/env python
"""The optimizer step on one H100, printed as one JSON line.  Writes nothing.

    python tools/bench_optim.py [--rounds 3] [--window-s 1.0] [--workloads filelist16,c2]

1. One optimizer step on the 34 M-parameter model's parameters (random gradients, norm above the clip so every path
   scales), device time from CUDA events, median of --rounds alternating windows:
     torch_foreach   clip_grad_norm_ + the reference's NoamOpt.step() over torch's foreach Adam (the reference loop)
     torch_fused     clip_grad_norm_ + torch Adam(fused=True)
     noam_step       NoamAdam.step() (no clip)
     noam_clip_step  NoamAdam.clip_and_step()
   with the bytes each step must move (from the shapes: read p, g, m, v and write p, m, v = 28 B per parameter, plus
   4 B per parameter for the norm pass where there is one) and the rate that gives.  The torch paths also read the norm
   on the host, as the reference loop's NaN guard does.
2. The full tf32 + flash-attention train step (tools/bench_train.py's workloads) with the reference's optimizer against
   clip_and_step, median of --rounds alternating windows.
The card name, power limit and max SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import importlib.util
import json
import math
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, REPO)

import torch  # noqa: E402

import bench_train as BT  # noqa: E402

REF_OPT = os.path.join(REPO, "oracle", "_ref", "core", "optimizer.py")
D_MODEL, WARMUP, FACTOR, CLIP = 384, 4000, 1.0, 1.0


def ref_optimizer():
    spec = importlib.util.spec_from_file_location("ref_core_optimizer", REF_OPT)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def windows(fns: dict, rounds: int, window_s: float) -> dict:
    for f in fns.values():
        f()
    torch.cuda.synchronize()
    per = {}
    for k, f in fns.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); f(); e1.record(); torch.cuda.synchronize()
        per[k] = e0.elapsed_time(e1)
    n = max(3, math.ceil(window_s * 1e3 / max(1e-3, min(per.values()))))
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                f()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / n)
    return {"iters_per_window": n, "ms": {k: sorted(v)[len(v) // 2] for k, v in ms.items()}, "ms_windows": ms}


def optimizer_step(R, rounds, window_s) -> dict:
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200 import optim as O
    from fastspeech2_b200.hparams import load_hp
    m = FeedForwardTransformer(68, 80, load_hp())
    m.load_state_dict(synthetic_state_dict(0), strict=True)
    base = [p.detach().to("cuda") for p in m.parameters()]
    n_params = sum(p.numel() for p in base)
    g = torch.Generator(device="cuda").manual_seed(0)
    grads = [torch.randn(p.shape, device="cuda", generator=g) * 1e-2 for p in base]

    def fresh():
        ps = [p.clone().requires_grad_() for p in base]
        for p, gr in zip(ps, grads):
            p.grad = gr.clone()
        return ps

    pf, pt, pn, pc = fresh(), fresh(), fresh(), fresh()
    ref = R.get_std_opt(types.SimpleNamespace(parameters=lambda: iter(pf)), D_MODEL, WARMUP, FACTOR)
    fused = torch.optim.Adam(pt, lr=1e-4, betas=(0.9, 0.98), eps=1e-9, fused=True)
    on = O.NoamAdam(pn, D_MODEL, FACTOR, WARMUP)
    oc = O.NoamAdam(pc, D_MODEL, FACTOR, WARMUP)

    def torch_foreach():
        gn = torch.nn.utils.clip_grad_norm_(pf, CLIP)
        if not math.isnan(gn):
            ref.step()

    def torch_fused():
        gn = torch.nn.utils.clip_grad_norm_(pt, CLIP)
        if not math.isnan(gn):
            fused.step()

    fns = {"torch_foreach": torch_foreach, "torch_fused": torch_fused, "noam_step": on.step,
           "noam_clip_step": lambda: oc.clip_and_step(CLIP)}
    out = windows(fns, rounds, window_s)
    moved = {"torch_foreach": 32, "torch_fused": 32, "noam_step": 28, "noam_clip_step": 32}
    out["params"] = n_params
    out["bytes_needed"] = {k: v * n_params for k, v in moved.items()}
    out["gb_per_s"] = {k: moved[k] * n_params / (out["ms"][k] * 1e-3) / 1e9 for k in fns}
    return out


def train_steps(R, name, rounds, window_s) -> dict:
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200 import optim as O
    from fastspeech2_b200.hparams import load_hp
    dev = torch.device("cuda")
    batch = BT.workload(name, dev)
    models = {}
    for kind in ("torch", "fused"):
        m = FeedForwardTransformer(68, 80, load_hp(), train_precision="tf32", train_attention="flash")
        m.load_state_dict(synthetic_state_dict(0), strict=True)
        m = m.to(dev).train()
        opt = O.get_std_opt(m, D_MODEL, WARMUP, FACTOR) if kind == "fused" else R.get_std_opt(m, D_MODEL, WARMUP, FACTOR)
        models[kind] = (m, opt)

    def step_torch():
        m, opt = models["torch"]
        loss, _ = m(*[batch[k] for k in BT.KEYS])
        loss.backward()
        gn = torch.nn.utils.clip_grad_norm_(m.parameters(), CLIP)
        if not math.isnan(gn):
            opt.step()
        opt.zero_grad()

    def step_fused():
        m, opt = models["fused"]
        loss, _ = m(*[batch[k] for k in BT.KEYS])
        loss.backward()
        opt.clip_and_step(CLIP)
        opt.zero_grad()

    out = windows({"torch": step_torch, "clip_and_step": step_fused}, rounds, window_s)
    out["B"], out["L"] = int(batch["xs"].shape[0]), int(batch["olens"].max())
    out["speedup"] = out["ms"]["torch"] / out["ms"]["clip_and_step"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window-s", type=float, default=1.0)
    ap.add_argument("--workloads", default="filelist16,c2")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    if not os.path.isfile(REF_OPT):
        raise SystemExit("the reference's core/optimizer.py is not staged in oracle/_ref (run build())")
    R = ref_optimizer()
    line = {"metric": "optimizer step (clip_grad_norm_ + Noam Adam) device ms, and the tf32 + flash train step with it",
            "card": BT.card(), "optimizer_step": optimizer_step(R, args.rounds, args.window_s)}
    torch.cuda.empty_cache()
    for name in [w for w in args.workloads.split(",") if w]:
        line[name] = train_steps(R, name, args.rounds, args.window_s)
        torch.cuda.empty_cache()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
