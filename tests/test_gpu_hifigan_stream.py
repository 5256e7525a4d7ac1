"""Windowed HiFi-GAN on the H100 (fs2_hifigan_window, `HiFiGANVocoder.window / stream / forward(chunk_frames=)`) against
the whole call, bit for bit, for V1 and V3 in every math mode: ragged per-utterance starts across the whole range, each
utterance alone, NaN outside a window's cone, the range check's halo rule, graph capture with starts rewritten in place,
chunked forward past fp32's whole-call limit, and the path from `synthesize`.  Weights as in test_gpu_hifigan.py (the
oracle's seeded init with every g moved away from |v|), mels ~ N(-6, 2^2)."""
import os

import numpy as np
import pytest
import torch

import _ups_window_plan as P
from conftest import GOLDEN
from fastspeech2_b200 import _lib
from fastspeech2_b200.hifigan import CONFIGS, HOP, HiFiGANVocoder
from oracle import hifigan_oracle as O

MODES = ["3xf16", "fp32", "f16", "tf32"]
CONFIG_NAMES = ["v1", "v3"]
OLENS = [37, 1, 300, 5, 160, 64, 301]
LAUNCHES = {"v1": 160, "v3": 49}                                    # the whole call's, fs2_hifigan, in every mode
N_FRAMES = [1, 2, 7, 13, 32, 100, 400]                              # 400 > Lmax


def _starts(kind, n):
    """Per-utterance starts (each utterance its own) of one category."""
    if kind == "zero":
        return [0] * len(OLENS)
    if kind == "halo":                                      # inside the left halo: the window clips at the utterance edge
        return [3, 0, 5, 1, 2, 6, 4]
    if kind == "interior":
        return [17, 0, 151, 2, 77, 29, 201]
    if kind == "end":                                       # olens - n .. olens: the core ends at olens
        return [max(0, o - n + b % 3) for b, o in enumerate(OLENS)]
    return [o + b % 2 * 50 for b, o in enumerate(OLENS)]   # "past": == olens and > olens, all-zero rows


KINDS = ["zero", "halo", "interior", "end", "past"]
CASES = [(k, n) for n in N_FRAMES for k in KINDS]


def check_coverage():
    """What the case table must reach for V1 and V3 (tests/test_hifigan_stream_args.py runs this without a GPU)."""
    missing = []
    for name in CONFIG_NAMES:
        cfg = P.hifigan(CONFIGS[name])
        U, h0 = len(cfg.rates), P.level_halo(cfg, 0)
        los = {}
        for kind, n in CASES:
            for s, o in zip(_starts(kind, n), OLENS):
                for buf, (lo, _) in P.windows(cfg, s, n, o).items():
                    los.setdefault(buf, set()).add(lo)
        for buf in [f"level{s}" for s in range(U + 1)] + [f"ups{s}" for s in range(U)]:
            if not any(lo % 128 for lo in los.get(buf, ())):
                missing.append(f"{name} {buf}: no start row off a 128-row tile boundary")
        # level s + 1 starts at u_s times ups s's start; ups s at c0 up_s - r_s, which only some levels can put off 16
        up = P.ups(cfg)
        for buf, allowed in [("level0", True)] + [(f"ups{s}", (up[s] % 16 or P.ups_reach(cfg, s) % 16) != 0) for s in range(U)]:
            if allowed and not any(lo % 16 for lo in los.get(buf, ())):
                missing.append(f"{name} {buf}: no start row off a 16-row boundary")
        starts = [(s, o, n) for kind, n in CASES for s, o in zip(_starts(kind, n), OLENS)]
        for what, pred in [("0", lambda s, o, n: s == 0), ("left halo", lambda s, o, n: 1 <= s <= h0 and s < o),
                           ("interior", lambda s, o, n: s > h0 and s + n < o - h0),
                           ("ends at olens", lambda s, o, n: s < o <= s + n and s > h0),
                           ("== olens", lambda s, o, n: s == o), ("> olens", lambda s, o, n: s > o)]:
            if not any(pred(*x) for x in starts):
                missing.append(f"{name}: no start {what}")
    if not any(n > max(OLENS) for _, n in CASES):
        missing.append("no n_frames above Lmax")
    return missing


pytestmark = pytest.mark.gpu


def _oracle(name, seed=0):
    torch.manual_seed(seed)
    g = O.Generator(CONFIGS[name])
    with torch.no_grad():
        for n, p in g.named_parameters():
            if n.endswith("weight_g"):
                p.mul_(torch.rand(p.shape) + 0.5)
    return g.eval()


@pytest.fixture(scope="module")
def case():
    gen = torch.Generator().manual_seed(1)
    mels = (torch.randn(len(OLENS), max(OLENS), 80, generator=gen) * 2 - 6).cuda()
    return {name: _oracle(name).state_dict() for name in CONFIG_NAMES}, mels, torch.tensor(OLENS).cuda()


@pytest.fixture(scope="module")
def vocoders(case):
    out = {}
    for name in CONFIG_NAMES:
        for m in MODES:
            v = HiFiGANVocoder(name, math_mode=m)
            v.load_state_dict(case[0][name])
            out[name, m] = v.cuda().eval()
    return out


@pytest.fixture(scope="module")
def whole(case, vocoders):
    _, mels, olens = case
    return {key: v(mels, olens)[0] for key, v in vocoders.items()}


def _expect(full, starts, n):
    """The window's expected audio: the whole call's samples, then +0."""
    B = full.shape[0]
    out = torch.zeros(B, n * HOP, device=full.device)
    for b, (s, o) in enumerate(zip(starts, OLENS)):
        k = max(0, min(n, o - s)) * HOP
        if k:
            out[b, :k] = full[b, s * HOP: s * HOP + k]
    return out


def _same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))          # +0 is +0, not -0


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", CONFIG_NAMES)
@pytest.mark.parametrize("n", N_FRAMES)
def test_window_is_the_whole_call_bit_for_bit(case, vocoders, whole, name, mode, n):
    _, mels, olens = case
    v = vocoders[name, mode]
    for kind in KINDS:
        starts = _starts(kind, n)
        audio, alens = v.window(mels, olens, torch.tensor(starts).cuda(), n)
        assert audio.shape == (len(OLENS), n * HOP)
        assert alens.tolist() == [max(0, min(n, o - s)) * HOP for s, o in zip(starts, OLENS)]
        assert _same_bits(audio, _expect(whole[name, mode], starts, n)), (name, mode, n, kind)
    # each utterance alone, B = 1, with host starts and its own Lmax
    starts = _starts("interior" if n < 100 else "end", n)
    audio, _ = v.window(mels, olens, starts, n)
    for b, (s, o) in enumerate(zip(starts, OLENS)):
        one, _ = v.window(mels[b: b + 1, :o].contiguous(), olens[b: b + 1], s, n)
        assert _same_bits(one[0], audio[b]), (name, mode, n, b)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", CONFIG_NAMES)
def test_nan_outside_the_cone_changes_nothing(case, vocoders, whole, name, mode):
    _, mels, olens = case
    v = vocoders[name, mode]
    h0 = v.window_plan()["halo"][0]
    for kind, n in (("interior", 7), ("halo", 13), ("end", 32)):
        starts = _starts(kind, n)
        nan = mels.clone()
        for b, (s, o) in enumerate(zip(starts, OLENS)):
            keep = torch.zeros(mels.shape[1], dtype=torch.bool)
            keep[max(0, s - h0): min(o, s + n + h0)] = True
            nan[b, ~keep] = float("nan")
        audio, _ = v.window(nan, olens, starts, n)                         # raises on any status bit
        assert _same_bits(audio, _expect(whole[name, mode], starts, n)), (name, mode, kind, n)
    if mode in ("3xf16", "f16"):                                           # a NaN that is read sets FS2_HIFIGAN_RANGE
        nan = mels.clone()
        nan[2, 151 - h0] = float("nan")
        with pytest.raises(ValueError, match="range"):
            v.window(nan, olens, _starts("interior", 7), 7)


@pytest.mark.parametrize("mode", ["3xf16", "f16"])
@pytest.mark.parametrize("name", CONFIG_NAMES)
def test_stream_concatenates_to_forward(case, vocoders, whole, name, mode):
    _, mels, olens = case
    v = vocoders[name, mode]
    for k in ((1, 5, 32, 333) if mode == "3xf16" else (32,)):
        chunks = list(v.stream(mels, olens, chunk_frames=k))
        assert len(chunks) == -(-max(OLENS) // k)
        audio = torch.cat([a for a, _ in chunks], 1)
        assert _same_bits(audio, whole[name, mode]), (name, mode, k)
        total = torch.stack([al for _, al in chunks]).sum(0)
        assert torch.equal(total, olens * HOP)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", CONFIG_NAMES)
def test_chunked_forward_is_forward(case, vocoders, whole, name, mode):
    _, mels, olens = case
    for k in (7, 64, 2000):
        audio, alens = vocoders[name, mode](mels, olens, chunk_frames=k)
        assert _same_bits(audio, whole[name, mode]) and torch.equal(alens, olens * HOP), (name, mode, k)


def test_chunked_fp32_runs_what_the_whole_call_refuses(case, vocoders):
    v = vocoders["v3", "fp32"]
    g = torch.Generator().manual_seed(5)
    big_olens = torch.randint(1, 902, (40,), generator=g)
    big_olens[3] = 901
    big = (torch.randn(40, 901, 80, generator=g) * 2 - 6).cuda()
    with pytest.raises(ValueError, match="fp32"):
        v(big, big_olens.cuda())
    audio, _ = v(big, big_olens.cuda(), chunk_frames=64)
    for lo in (0, 20):                                                     # sub-batches the whole call accepts
        part, _ = v(big[lo: lo + 20], big_olens[lo: lo + 20].cuda())
        assert _same_bits(audio[lo: lo + 20], part), lo


def _raw_window(v, mels, olens, starts, n, audio, status, ws):
    dev = mels.device
    _lib.check(_lib.load().fs2_hifigan_window(v._handle(dev), _lib.ptr(mels), _lib.ptr(olens), _lib.ptr(starts), mels.shape[0],
                                              mels.shape[1], n, _lib.ptr(audio), audio.shape[1], _lib.ptr(status), _lib.ptr(ws), ws.numel(),
                                              _lib.stream_ptr(dev)), "fs2_hifigan_window")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", CONFIG_NAMES)
def test_graph_replay_with_rewritten_starts(case, vocoders, name, mode):
    _, mels, olens = case
    v = vocoders[name, mode]
    n = 13
    B = mels.shape[0]
    starts = torch.zeros(B, dtype=torch.int64, device="cuda")
    audio = torch.empty(B, n * HOP, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    ws = v._window_workspace(v._handle(mels.device), B, n, mels.device)
    lib = _lib.load()
    before = lib.fs2_kernel_launches()
    _raw_window(v, mels, olens, starts, n, audio, status, ws)
    assert lib.fs2_kernel_launches() - before == LAUNCHES[name] == v.launches()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _raw_window(v, mels, olens, starts, n, audio, status, ws)
    for kind in KINDS:
        st = _starts(kind, n)
        starts.copy_(torch.tensor(st))
        audio.fill_(7.0)
        graph.replay()
        torch.cuda.synchronize()
        assert int(status.item()) == 0
        eager, _ = v.window(mels, olens, st, n)
        assert _same_bits(audio, eager), (name, mode, kind)
    starts.copy_(torch.tensor([0, -1, 0, 0, 0, 0, 0]))
    graph.replay()
    assert int(status.item()) == _lib.FS2_HIFIGAN_BAD_START
    assert torch.all(audio[1].view(torch.int32) == 0)
    with pytest.raises(ValueError, match="starts"):
        v.window(mels, olens, starts, n)


@pytest.mark.parametrize("name", CONFIG_NAMES)
def test_range_is_raised_exactly_for_windows_whose_cone_holds_the_spike(case, vocoders, whole, name):
    sds, mels, olens = case
    f = 150                                                  # utterance 2 (300 frames)
    spiked = mels.clone()
    spiked[2, f] = 1e5                                       # far above 4094 in the mel operand
    n = 13
    for mode in ("3xf16", "f16"):
        v = vocoders[name, mode]
        h0 = v.window_plan()["halo"][0]
        with pytest.raises(ValueError, match="range"):
            v(spiked, olens)
        with pytest.raises(ValueError, match="range"):                   # chunked: the whole call's status
            v(spiked, olens, chunk_frames=32)
        for s in (f - h0 - n, f - h0 - n + 1, f - n, f, f + h0, f + h0 + 1, 250):
            starts = [0, 0, s, 0, 0, 0, 0]
            if s - h0 <= f < s + n + h0:
                with pytest.raises(ValueError, match="range"):
                    v.window(spiked, olens, starts, n)
            else:
                audio, _ = v.window(spiked, olens, starts, n)
                assert _same_bits(audio, _expect(whole[name, mode], starts, n)), (name, mode, s)
    sd = dict(sds[name])
    sd["conv_pre.weight_g"] = sd["conv_pre.weight_g"] * 3e4      # conv_pre's output far beyond 4094
    for mode in ("f16", "3xf16", "fp32"):
        v = HiFiGANVocoder(name, math_mode=mode)
        v.load_state_dict(sd)
        v = v.cuda()
        if mode == "fp32":
            audio, _ = v.window(mels, olens, 100, n)
            assert torch.isfinite(audio).all()
        else:
            with pytest.raises(ValueError, match="range"):
                v.window(mels, olens, 100, n)


def test_end_to_end_stream_after_synthesize():
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.hparams import load_hp
    model = FeedForwardTransformer(68, 80, load_hp())
    model.load_state_dict(synthetic_state_dict(0), strict=True)
    model = model.cuda().eval()
    fl = np.load(os.path.join(GOLDEN, "filelist64.npz"))
    with torch.no_grad():
        mels, olens, _ = model.synthesize(torch.from_numpy(fl["xs"]).cuda(), torch.from_numpy(fl["ilens"]).cuda())
    v = HiFiGANVocoder("v3").cuda()
    want, _ = v(mels, olens)
    got = torch.cat([a for a, _ in v.stream(mels, olens, chunk_frames=32)], 1)
    assert _same_bits(got, want)
    chunked, _ = v(mels, olens, chunk_frames=64)
    assert _same_bits(chunked, want)
