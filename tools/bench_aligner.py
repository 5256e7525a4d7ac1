#!/usr/bin/env python
"""The duration aligner on one H100 (fastspeech2_b200.aligner), printed as one JSON line.  Writes nothing in the tree.

    python tools/bench_aligner.py [--steps 20] [--rounds 3]

Workload: the 1,024 utterances of tests/golden/align_filelist.npz (LJSpeech phoneme strings and MFA durations) rendered
as a synthetic corpus (tests/_aligner_corpus.py); train batches are B = 32 from the same length-bucketed sampler as
`train`.  Device events around `--steps` calls, median of `--rounds` windows:
  train_step_ms    forward, backward and clip_and_step of one batch with the binarization loss on (what a step after
                   bin_start costs), cycling through 8 fixed batches
  split_ms         the same batches' parts alone: convolutions (keys and queries, forward and backward), logprob
                   (forward and backward), forward_sum (forward, then backward with dlogp), mas, bin_loss (forward and
                   backward)
  extract          Aligner.durations over the whole corpus in B = 32 batches, host batching included, in utterances/s
The card name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from _aligner_corpus import fixture_lines, render  # noqa: E402
from bench_features import timed  # noqa: E402
from bench_per_utterance import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_aligner needs a CUDA device")
    from fastspeech2_b200 import aligner as A
    from fastspeech2_b200.data import BucketBatchSampler

    lines = fixture_lines()
    sym = A.build_symbols(lines)
    corpus = A.Corpus(lines, sym, mels=render(lines, 0))
    torch.manual_seed(0)
    model = A.Aligner(len(sym)).cuda()
    opt = A.NoamAdam(model.parameters(), A.EMB, 1.0, 4000)
    batches = [corpus.batch(idx, "cuda") for idx in list(BucketBatchSampler(corpus.frames, 32, seed=0))[:8]]
    shapes = [(int(b[0].shape[1]), int(b[2].shape[1])) for b in batches]
    it = iter(range(1 << 30))

    def step():
        b = batches[next(it) % len(batches)]
        loss, *_ = model.loss(*b, bin_weight=1.0)
        opt.zero_grad()
        loss.backward()
        opt.clip_and_step(1.0)
    res = {"workload": "align_filelist synthetic, B = 32", "batches_T_L": shapes,
           "train_step_ms": round(timed(step, args.steps, args.rounds), 3)}

    st = torch.zeros(7, dtype=torch.int32, device="cuda")
    prep = []
    for b in batches:
        xs, il, mels, ol = A.Aligner._inputs(*b)
        with torch.no_grad():
            k, q = model.keys_queries(xs, il, mels, ol)
            logp = A.AlignLogProbFn.apply(q, k, il, ol, st)
            _, path = A.mas(logp, il, ol, st)
        prep.append((xs, il, mels, ol, q, k, logp, path))
    cyc = iter(range(1 << 30))

    def nxt():
        return prep[next(cyc) % len(prep)]

    def convs():
        xs, il, mels, ol, *_ = nxt()
        k, q = model.keys_queries(xs, il, mels, ol)
        torch.autograd.backward([k, q], [torch.ones_like(k), torch.ones_like(q)])

    def logprob():
        _, il, _, ol, q, k, *_ = nxt()
        q, k = q.detach().requires_grad_(True), k.detach().requires_grad_(True)
        lp = A.AlignLogProbFn.apply(q, k, il, ol, st)
        lp.backward(torch.ones_like(lp))

    def forward_sum():
        _, il, _, ol, _, _, logp, _ = nxt()
        lp = logp.detach().requires_grad_(True)
        A.ForwardSumFn.apply(lp, il, ol, st).sum().backward()

    def mas():
        _, il, _, ol, _, _, logp, _ = nxt()
        A.mas(logp, il, ol, st)

    def bin_loss():
        _, il, _, ol, _, _, logp, path = nxt()
        lp = logp.detach().requires_grad_(True)
        A.BinLossFn.apply(lp, path, il, ol, st).sum().backward()
    res["split_ms"] = {k: round(timed(fn, args.steps, args.rounds), 3) for k, fn in
                       (("convolutions", convs), ("logprob", logprob), ("forward_sum", forward_sum), ("mas", mas), ("bin_loss", bin_loss))}
    A.extract(model, corpus)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    A.extract(model, corpus)
    torch.cuda.synchronize()
    res["extract"] = {"utterances": len(corpus.lines), "utt_per_s": round(len(corpus.lines) / (time.perf_counter() - t0), 1)}
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
