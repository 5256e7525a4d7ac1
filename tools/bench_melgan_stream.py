#!/usr/bin/env python
"""Streamed MelGAN (`MelGANVocoder.window / stream / forward(chunk_frames=)`) on one H100, printed as one JSON line.
Writes nothing.

    python tools/bench_melgan_stream.py [--steps 2] [--rounds 3]

Workloads: the mels `synthesize` returns for the 64 sequences of tests/golden/filelist64.npz (seeded random weights:
only the lengths matter for time), and the same frames concatenated into one [1, sum(olens), 80] paragraph, as
inference.py vocodes them.  Per math mode (3xf16, f16) and window size n_frames (16, 32, 64):
  first_audio_ms    CUDA events from enqueue to completion of the first window (frames [0, n) of every utterance), beside
                    the whole call (`forward`), whose first sample is ready only when it ends;
  stream_ms         a full lockstep stream of windows (Lmax / n calls, the window's C entry on preallocated buffers) against
                    one `forward`: the measured overhead, beside the FLOP overhead counted from the window shapes;
  graph / eager     at B = 1, where launches dominate: one window call eager against one replay of a captured graph;
  fp32_chunked      `forward(chunk_frames=64)` in fp32 on filelist64, which the whole call refuses (B * (Lmax + 10) * 256
                    above 65535 * 128);
  workspace_bytes   of each row's call.
Timed variants run in alternating windows of `--steps` calls, median of `--rounds` windows.  Before timing, the streamed
audio is asserted equal to `forward`'s bit for bit wherever the whole call runs.  The card name, power limit and max SM
clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_per_utterance import alternate, card, median  # noqa: E402

HOP = 256
N_FRAMES = (16, 32, 64)


def max_sm_clock():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=20)
        return r.stdout.strip() or None
    except Exception:
        return None


class Stream:
    """Preallocated lockstep windows of one batch: starts for every step on the device, one output row block per step."""

    def __init__(self, voc, mels, olens, n):
        self.voc, self.mels, self.olens, self.n = voc, mels.contiguous(), olens.contiguous(), n
        B, L = mels.shape[:2]
        self.B, self.L = B, L
        dev = mels.device
        self.h = voc._handle(dev)
        self.ws = voc._window_workspace(self.h, B, n, dev)
        self.steps = -(-L // n)
        self.starts = (torch.arange(self.steps, device=dev, dtype=torch.int64) * n)[:, None].expand(self.steps, B).contiguous()
        self.audio = torch.empty(B, self.steps * n * HOP, device=dev)
        self.status = torch.zeros(self.steps, dtype=torch.int32, device=dev)

    def window(self, k):
        self.voc._window_call(self.h, self.mels, self.olens, self.starts[k], self.B, self.L, self.n, self.audio[:, k * self.n * HOP:],
                              self.steps * self.n * HOP, self.status[k: k + 1], self.ws)

    def run(self):
        for k in range(self.steps):
            self.window(k)


def event_ms(fn, rounds):
    """Median of `rounds` event-timed calls of fn (enqueue to completion), after one warm-up call."""
    out = []
    fn()
    for _ in range(rounds):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return median(out), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import _ups_window_plan as P
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.hparams import load_hp
    from fastspeech2_b200.melgan import MelGANVocoder
    from oracle.melgan_oracle import Generator

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
    para_olens = torch.tensor([para.shape[1]], device=dev)
    workloads = {"filelist64": (mels.contiguous(), olens), "paragraph": (para, para_olens)}

    torch.manual_seed(0)
    gen = Generator().eval()
    voc = {}
    for m in ("3xf16", "f16", "fp32"):
        voc[m] = MelGANVocoder(math_mode=m)
        voc[m].load_state_dict(gen.state_dict())
        voc[m] = voc[m].to(dev).eval()

    def ws_bytes(v, B, n=None, L=None):
        import ctypes as C
        from fastspeech2_b200 import _lib
        out = C.c_size_t()
        h = v._handle(dev)
        if n is None:
            _lib.check(_lib.load().fs2_melgan_workspace_bytes(h, B, L, C.byref(out)), "ws")
        else:
            _lib.check(_lib.load().fs2_melgan_window_workspace_bytes(h, B, n, C.byref(out)), "ws")
        return out.value

    rows = []
    bit_identical = True
    with torch.no_grad():
        for mode in ("3xf16", "f16"):
            v = voc[mode]
            for wname, (m, o) in workloads.items():
                B, L = m.shape[:2]
                whole, _ = v(m, o)
                whole_ms, whole_w = event_ms(lambda: v(m, o), args.rounds)
                for n in N_FRAMES:
                    s = Stream(v, m, o, n)
                    s.run()
                    torch.cuda.synchronize()
                    assert int(s.status.abs().sum()) == 0
                    same = torch.equal(s.audio[:, : L * HOP].view(torch.int32), whole.view(torch.int32))
                    assert same, (mode, wname, n)
                    bit_identical &= same
                    first_ms, first_w = event_ms(lambda: s.window(0), args.rounds)
                    row = {"mode": mode, "workload": wname, "B": B, "Lmax": L, "n_frames": n, "windows": s.steps,
                           "first_audio_ms": first_ms, "first_audio_ms_windows": first_w, "whole_call_ms": whole_ms,
                           "whole_call_ms_windows": whole_w, "window_workspace_bytes": ws_bytes(v, B, n),
                           "whole_call_workspace_bytes": ws_bytes(v, B, L=L),
                           "flop_overhead_from_shapes": P.window_flop_overhead(P.melgan(), n)}
                    # a full stream over the paragraph at n = 16 is ~2300 calls: timed at n = 64 only
                    if wname == "filelist64" or n == 64:
                        t = alternate({"stream": s.run, "forward": lambda: v(m, o)}, args.steps, args.rounds)
                        row.update({"stream_ms": median(t["stream"]), "stream_ms_windows": t["stream"],
                                    "forward_ms": median(t["forward"]), "forward_ms_windows": t["forward"],
                                    "stream_overhead_measured": median(t["stream"]) / median(t["forward"]) - 1})
                    rows.append(row)
                    del s

            # B = 1 eager against graph replay: one window of 32 frames at an interior start of the paragraph
            m, o = workloads["paragraph"]
            s = Stream(v, m, o, 32)
            k = s.steps // 2
            s.audio.zero_()
            s.window(k)
            torch.cuda.synchronize()
            ref = s.audio.clone()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                s.window(k)
            s.audio.zero_()
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(ref.view(torch.int32), s.audio.view(torch.int32))
            t = alternate({"eager": lambda: s.window(k), "graph": g.replay}, max(args.steps, 20), args.rounds)
            rows.append({"mode": mode, "workload": "paragraph B=1 window", "n_frames": 32, "eager_ms": median(t["eager"]),
                         "eager_ms_windows": t["eager"], "graph_ms": median(t["graph"]), "graph_ms_windows": t["graph"],
                         "window_workspace_bytes": ws_bytes(v, 1, 32)})
            del s, g

        # fp32: the whole call refuses filelist64; chunked forward runs it with one window's workspace
        m, o = workloads["filelist64"]
        v = voc["fp32"]
        try:
            v(m, o)
            refused = False
        except ValueError:
            refused = True
        t = alternate({"fp32_chunked": lambda: v(m, o, chunk_frames=64)}, args.steps, args.rounds)
        rows.append({"mode": "fp32", "workload": "filelist64 forward(chunk_frames=64)", "whole_call_refused": refused,
                     "ms": median(t["fp32_chunked"]), "ms_windows": t["fp32_chunked"], "window_workspace_bytes": ws_bytes(v, m.shape[0], 64)})

    info = card()
    info["max_sm_clock"] = max_sm_clock()
    line = {"metric": "streamed MelGAN: time to first audio, stream overhead, fp32 chunked", "card": info,
            "filelist64_valid_frames": sum(ol), "paragraph_frames": int(para.shape[1]), "streamed_equals_forward_bitwise": bit_identical,
            "rows": rows, "timing_note": f"alternating windows of {args.steps} calls, median of {args.rounds} windows; first audio and whole "
                                         f"call: median of {args.rounds} event-timed calls"}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
