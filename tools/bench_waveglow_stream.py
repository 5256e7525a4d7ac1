#!/usr/bin/env python
"""Streamed WaveGlow (`WaveGlowVocoder.window / stream`) on one H100, printed as one JSON line.  Writes nothing.

    python tools/bench_waveglow_stream.py [--steps 1] [--rounds 1] [--channels 256,512]

Workloads: the mels `synthesize` returns for the 64 sequences of tests/golden/filelist64.npz (seeded random weights:
only the lengths matter for time), and the same frames concatenated into one [1, sum(olens), 80] paragraph.  Seeded
random WaveGlow weights at n_channels C = 256 and 512, sigma 0.6, seed 0.  Per C, math mode (3xf16, f16), workload and
window size n_frames (32, 64, 128):
  first_audio_ms    CUDA events from enqueue to completion of the first window (frames [0, n) of every utterance), beside
                    the whole call (`forward`), whose first sample is ready only when it ends;
  stream_ms         a full lockstep stream of windows (ceil(Lmax / n) calls of the window's C entry on preallocated
                    buffers) against one `forward`, alternated: the measured overhead, beside the FLOP overhead counted
                    from the buffer shapes (FLOP_OVERHEAD_NOTE).  Timed at C = 256 and n = 128 only (a filelist64
                    stream at C = 512 takes tens of seconds); every timed stream is first asserted equal to `forward`
                    bit for bit;
  graph / eager     at B = 1, where launches dominate: one 32-frame window at an interior start of the paragraph, eager
                    against one replay of a captured graph;
  workspace_bytes   of the window and of the whole call.
The card name, power limit and max SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_melgan_stream import event_ms, max_sm_clock  # noqa: E402
from bench_per_utterance import alternate, card, median  # noqa: E402

HOP = 256
N_FRAMES = (32, 64, 128)
SEED, SIGMA = 0, 0.6
FLOP_OVERHEAD_NOTE = ("window FLOP over the whole call's, from shapes: every GEMM is linear in rows and a window computes "
                      "its buffer's frames [max(0, s - 96), min(olens, s + n + 96)) per utterance")


class Stream:
    """Preallocated lockstep windows of one batch: starts for every step on the device, one output row block per step."""

    def __init__(self, voc, mels, olens, n, seeds):
        self.mels, self.olens, self.n = mels.contiguous(), olens.contiguous(), n
        B, L = mels.shape[:2]
        self.B, self.L = B, L
        dev = mels.device
        self.h = voc._handle(dev)
        self.ws = voc._window_workspace(self.h, B, n, dev)
        self.call = voc._window_call(SIGMA, seeds, None)
        self.steps = -(-L // n)
        self.starts = (torch.arange(self.steps, device=dev, dtype=torch.int64) * n)[:, None].expand(self.steps, B).contiguous()
        self.audio = torch.empty(B, self.steps * n * HOP, device=dev)
        self.status = torch.zeros(self.steps, dtype=torch.int32, device=dev)

    def window(self, k):
        self.call(self.h, self.mels, self.olens, self.starts[k], self.B, self.L, self.n, self.audio[:, k * self.n * HOP:],
                  self.steps * self.n * HOP, self.status[k: k + 1], self.ws)

    def run(self):
        for k in range(self.steps):
            self.window(k)


def buffer_frames(ol, n, L):
    """Frames every window of a lockstep stream computes, summed over the stream (empty windows compute none)."""
    import _waveglow_window_plan as P
    total = 0
    for s in range(0, L, n):
        for o in ol:
            w = P.buffer(s, min(n, L - s), o)
            if w is not None:
                total += w[1] - w[0]
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--channels", default="256,512")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from fastspeech2_b200 import FeedForwardTransformer, _lib, synthetic_state_dict
    from fastspeech2_b200.hparams import load_hp
    from fastspeech2_b200.waveglow import WaveGlowVocoder
    from oracle import waveglow_oracle as O

    dev = torch.device("cuda", torch.cuda.current_device())
    model = FeedForwardTransformer(68, 80, load_hp(), precision="3xf16")
    model.load_state_dict(synthetic_state_dict(0), strict=True)
    model = model.to(dev).eval()
    fl = np.load(os.path.join(ROOT, "tests", "golden", "filelist64.npz"))
    with torch.no_grad():
        mels, olens, _ = model.synthesize(torch.from_numpy(fl["xs"]).to(dev), torch.from_numpy(fl["ilens"]).to(dev))
    del model
    ol = [int(v) for v in olens.tolist()]
    para = torch.cat([mels[b, :n] for b, n in enumerate(ol)], 0)[None].contiguous()        # [1, sum(olens), 80]
    workloads = {"filelist64": (mels.contiguous(), olens, ol), "paragraph": (para, torch.tensor([para.shape[1]], device=dev), [para.shape[1]])}

    def ws_bytes(v, B, n=None, L=None):
        out = C.c_size_t()
        h = v._handle(dev)
        if n is None:
            _lib.check(_lib.load().fs2_waveglow_workspace_bytes(h, B, L, C.byref(out)), "ws")
        else:
            _lib.check(_lib.load().fs2_waveglow_window_workspace_bytes(h, B, n, C.byref(out)), "ws")
        return out.value

    rows = []
    bit_identical = True
    with torch.no_grad():
        for Cn in [int(c) for c in args.channels.split(",")]:
            torch.manual_seed(0)
            g = O.WaveGlow(Cn).eval()
            for mode in ("3xf16", "f16"):
                v = WaveGlowVocoder(n_channels=Cn, math_mode=mode)
                v.load_state_dict(g.state_dict())
                v = v.to(dev).eval()
                for wname, (m, o, lens) in workloads.items():
                    B, L = m.shape[:2]
                    seeds = v._seeds(SEED, B, dev)
                    fwd = lambda: v(m, o, sigma=SIGMA, seed=seeds)
                    whole, _ = fwd()
                    whole_ms, whole_w = event_ms(fwd, args.rounds)
                    whole_ws = ws_bytes(v, B, L=L)
                    v._ws.clear()                                   # the whole call's workspace is tens of GB at C = 512
                    torch.cuda.empty_cache()
                    for n in N_FRAMES:
                        s = Stream(v, m, o, n, seeds)
                        first_ms, first_w = event_ms(lambda: s.window(0), args.rounds)
                        row = {"C": Cn, "mode": mode, "workload": wname, "B": B, "Lmax": L, "n_frames": n, "windows": s.steps,
                               "first_audio_ms": first_ms, "first_audio_ms_windows": first_w, "whole_call_ms": whole_ms,
                               "whole_call_ms_windows": whole_w, "window_workspace_bytes": ws_bytes(v, B, n),
                               "whole_call_workspace_bytes": whole_ws,
                               "flop_overhead_from_shapes": buffer_frames(lens, n, L) / sum(lens) - 1}
                        if Cn == 256 and n == 128:
                            s.run()
                            torch.cuda.synchronize()
                            assert int(s.status.abs().sum()) == 0
                            same = torch.equal(s.audio[:, : L * HOP].view(torch.int32), whole.view(torch.int32))
                            assert same, (Cn, mode, wname, n)
                            bit_identical &= same
                            t = alternate({"stream": s.run, "forward": fwd}, args.steps, args.rounds)
                            row.update({"stream_ms": median(t["stream"]), "stream_ms_windows": t["stream"],
                                        "forward_ms": median(t["forward"]), "forward_ms_windows": t["forward"],
                                        "stream_overhead_measured": median(t["stream"]) / median(t["forward"]) - 1})
                            v._ws.clear()
                        rows.append(row)
                        del s
                        v._wws.clear()
                        torch.cuda.empty_cache()
                    del whole

                # B = 1 eager against graph replay: one window of 32 frames at an interior start of the paragraph
                m, o, _ = workloads["paragraph"]
                s = Stream(v, m, o, 32, v._seeds(SEED, 1, dev))
                k = s.steps // 2
                s.audio.zero_()
                s.window(k)
                torch.cuda.synchronize()
                ref = s.audio.clone()
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr):
                    s.window(k)
                s.audio.zero_()
                gr.replay()
                torch.cuda.synchronize()
                assert torch.equal(ref.view(torch.int32), s.audio.view(torch.int32))
                t = alternate({"eager": lambda: s.window(k), "graph": gr.replay}, max(args.steps, 10), args.rounds + 1)
                rows.append({"C": Cn, "mode": mode, "workload": "paragraph B=1 window", "n_frames": 32, "eager_ms": median(t["eager"]),
                             "eager_ms_windows": t["eager"], "graph_ms": median(t["graph"]), "graph_ms_windows": t["graph"],
                             "window_workspace_bytes": ws_bytes(v, 1, 32)})
                del s, gr, v
                torch.cuda.empty_cache()

    info = card()
    info["max_sm_clock"] = max_sm_clock()
    line = {"metric": "streamed WaveGlow: time to first audio, stream overhead, graph replay, workspace", "card": info,
            "filelist64_valid_frames": sum(ol), "paragraph_frames": int(para.shape[1]), "streamed_equals_forward_bitwise": bit_identical,
            "flop_overhead_note": FLOP_OVERHEAD_NOTE, "rows": rows,
            "timing_note": f"stream / forward: alternating windows of {args.steps} calls, median of {args.rounds} windows; first audio "
                           f"and whole call: median of {args.rounds} event-timed calls after a warm-up call"}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
