#!/usr/bin/env python
"""External speaker embeddings (DESIGN.md section 27) on one H100, printed as one JSON line.  Writes nothing in the tree.

    python tools/bench_spembs.py [--steps 10] [--rounds 5]

Device events around `--steps` calls, median of `--rounds` windows; each pair of arms alternates window by window:
  synthesize_ms   `synthesize` at B = 64 on LJSpeech-shaped input (T = 100 phonemes, 3xf16): the model without embeddings
                  against the same weights with a zero 512-dim projection, so that both arms predict the same durations
                  and decode the same frames (the add is fused into the last encoder LayerNorm; the projection is one
                  extra launch)
  train_step_ms   a TF32 train step (forward + backward) at B = 16 and B = 64, T = 100, L = 800, without and with 512-dim
                  embeddings
  project_ms      fs2_spemb_project and fs2_spemb_project_backward alone at B = 64, adim = 256, D in {192, 512}
The card name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench_per_utterance import card  # noqa: E402
from bench_speakers import paired  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_spembs needs a CUDA device")
    from fastspeech2_b200 import FeedForwardTransformer, _lib
    from fastspeech2_b200.hparams import load_hp
    from fastspeech2_b200.synthetic import make_batch
    from fastspeech2_b200.weights import synthetic_state_dict

    sd = synthetic_state_dict(7)
    D = 512
    g = torch.Generator().manual_seed(1)
    W, bias = torch.randn(256, D, generator=g) * 0.5, torch.randn(256, generator=g) * 0.1

    def model(d, zero=False, **kw):
        hp = load_hp()
        hp["model"]["spk_embed_dim"] = d
        m = FeedForwardTransformer(68, 80, hp, **kw)
        w = dict(sd)
        if d:
            w["spk_embed_proj.weight"] = torch.zeros(256, d) if zero else W
            w["spk_embed_proj.bias"] = torch.zeros(256) if zero else bias
        m.load_state_dict(w, strict=True)
        return m.cuda()

    res = {"workload": "LJSpeech-shaped synthetic, T = 100, L = 800", "D": D}
    # (a) synthesize, B = 64, 3xf16
    plain, spe = model(0, precision="3xf16").eval(), model(D, zero=True, precision="3xf16").eval()
    bt = make_batch(64, 100, 800, seed=3, ilens=[100 - (b % 37) for b in range(64)])
    xs, il = bt["xs"].cuda(), bt["ilens"].cuda()
    e = torch.randn(64, D, generator=torch.Generator().manual_seed(2)).cuda()
    with torch.no_grad():
        a, b = paired([lambda: plain.synthesize(xs, il), lambda: spe.synthesize(xs, il, spembs=e)], args.steps, args.rounds)
        frames = int(plain.synthesize(xs, il)[1].sum())
    res["synthesize_ms"] = {"B": 64, "precision": "3xf16", "frames": frames, "plain": a, "spembs": b}
    del plain, spe
    # (b) TF32 train step
    res["train_step_ms"] = {}
    for B in (16, 64):
        plain, spe = model(0, train_precision="tf32").train(), model(D, train_precision="tf32").train()
        tb = make_batch(B, 100, 800, seed=B)
        args_ = [tb[k].cuda() for k in ("xs", "ilens", "ys", "olens", "ds", "es", "ps")]
        eb = e[:B].contiguous()

        def step(m, **kw):
            loss, _ = m(*args_, **kw)
            loss.backward()
            for p in m.parameters():
                p.grad = None
        a, b = paired([lambda: step(plain), lambda: step(spe, spembs=eb)], max(1, args.steps // 2), args.rounds)
        res["train_step_ms"][f"B={B}"] = {"plain": a, "spembs": b}
        del plain, spe
    # (c) the projection and its backward alone
    lib = _lib.load()
    st = _lib.stream_ptr(e.device)
    res["project_ms"] = {}
    for d in (192, 512):
        Wd, bd = torch.randn(256, d, device="cuda"), torch.randn(256, device="cuda")
        ed = torch.randn(64, d, device="cuda")
        v, en = torch.empty(64, 256, device="cuda"), torch.empty(64, d, device="cuda")
        dv, dW, db = torch.randn(64, 256, device="cuda"), torch.zeros(256, d, device="cuda"), torch.zeros(256, device="cuda")
        fwd = lambda: lib.fs2_spemb_project(Wd.data_ptr(), bd.data_ptr(), ed.data_ptr(), 64, d, 256, v.data_ptr(), en.data_ptr(),
                                            None, None, st)
        bwd = lambda: lib.fs2_spemb_project_backward(dv.data_ptr(), en.data_ptr(), 64, d, 256, dW.data_ptr(), db.data_ptr(), st)
        f, b = paired([fwd, bwd], 200, args.rounds)
        res["project_ms"][f"D={d}"] = {"forward": f, "backward": b}
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
