"""Windowed WaveGlow on the H100 (fs2_waveglow_window, `WaveGlowVocoder.window / stream / forward(chunk_frames=)`)
against the whole call, bit for bit, in every math mode: ragged per-utterance starts at both utterance edges, one edge
and the interior, seeds and z, reversed batch order, NaN outside a window's cone, the range check's halo rule, graph
capture with starts rewritten in place and the launch count, chunked fp32 past the whole call's limit, and the path from
`synthesize`.  Weights as in test_gpu_waveglow.py (make_oracle), mels ~ N(-6, 2^2)."""
import os

import numpy as np
import pytest
import torch

import _waveglow_window_plan as P
from conftest import GOLDEN
from fastspeech2_b200 import _lib
from fastspeech2_b200.waveglow import HOP, STEPS, WaveGlowVocoder

MODES = ["3xf16", "fp32", "f16", "tf32"]
OLENS = [420, 1, 37, 300, 5, 262]
N_FRAMES = [1, 7, 32, 64, 128]
LAUNCHES = {"3xf16": 498, "f16": 498, "tf32": 497, "fp32": 497}     # fs2_waveglow's and the audio copy


def _starts(kind, n):
    """Per-utterance starts (each utterance its own) of one category."""
    if kind == "zero":
        return [0] * len(OLENS)
    if kind == "left":                                      # inside the left halo: the buffer starts at the utterance edge
        return [3, 0, 5, 50, 2, 90]
    if kind == "interior":                                  # buffers off the utterance edge, first rows at every residue
        return [97 + n % 4, 0, 10, 98 + n % 3, 1, 99]
    if kind == "end":                                       # olens - n .. olens: the core ends at olens
        return [max(0, o - n + b % 3) for b, o in enumerate(OLENS)]
    return [o + b % 2 * 50 for b, o in enumerate(OLENS)]   # "past": == olens and > olens, all-zero rows


KINDS = ["zero", "left", "interior", "end", "past"]
CASES = [(k, n) for n in N_FRAMES for k in KINDS]


def check_coverage():
    """What the case table must reach (tests/test_waveglow_stream_args.py runs this without a GPU)."""
    missing = []
    bufs = [(s, o, n, P.buffer(s, n, o)) for kind, n in CASES for s, o in zip(_starts(kind, n), OLENS)]
    live = [(s, o, n, w) for s, o, n, w in bufs if w is not None]
    for what, pred in [("both edges", lambda f0, f1, o: f0 == 0 and f1 == o), ("left edge only", lambda f0, f1, o: f0 == 0 and f1 < o),
                       ("right edge only", lambda f0, f1, o: f0 > 0 and f1 == o),
                       ("interior with full halos", lambda f0, f1, o: f0 > 0 and f1 < o)]:
        if not any(pred(w[0], w[1], o) for _, o, _, w in live):
            missing.append(f"no window at {what}")
    if not any(o > n + 2 * P.halo() and w[0] > 0 and w[1] < o for _, o, n, w in live):
        missing.append("no interior window of an utterance longer than n + 192 frames")
    if not any(s == o for s, o, _, _ in bufs) or not any(s > o for s, o, _, _ in bufs):
        missing.append("no start at and past olens")
    residues = {w[0] * STEPS % 128 for _, _, _, w in live if w[0] > 0}
    if residues != {0, 32, 64, 96}:
        missing.append(f"buffer first rows reach only the residues {sorted(residues)} mod 128")
    if not any((w[1] - w[0]) * STEPS % 128 for _, _, _, w in live):
        missing.append("no ragged buffer tail")
    return missing


pytestmark = pytest.mark.gpu
DEV = "cuda"


def _vocoder(g, mode):
    from test_gpu_waveglow import vocoder
    return vocoder(g, mode)


def _bits(t):
    return t.contiguous().view(torch.int32)                  # +0 is +0, not -0


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


def _expect(full, olens, starts, n):
    """The window's expected audio: the whole call's samples, then +0."""
    out = torch.zeros(full.shape[0], n * HOP, device=full.device)
    for b, (s, o) in enumerate(zip(starts, olens)):
        k = max(0, min(n, o - s)) * HOP
        if k:
            out[b, :k] = full[b, s * HOP: s * HOP + k]
    return out


@pytest.fixture(scope="module")
def case():
    from test_gpu_waveglow import make_oracle
    g = make_oracle(64, 0)
    gen = torch.Generator().manual_seed(1)
    B, L = len(OLENS), max(OLENS)
    mels = (torch.randn(B, L, 80, generator=gen) * 2 - 6).to(DEV)
    z = torch.randn(B, 8, L * STEPS, generator=gen).to(DEV)
    seeds = torch.arange(40, 40 + B, device=DEV)
    return g, mels, torch.tensor(OLENS, device=DEV), z, seeds


@pytest.fixture(scope="module")
def vocoders(case):
    return {m: _vocoder(case[0], m) for m in MODES}


@pytest.fixture(scope="module")
def whole(case, vocoders):
    _, mels, olens, z, seeds = case
    return {m: {"seed": vocoders[m](mels, olens, seed=seeds, sigma=0.8)[0], "z": vocoders[m](mels, olens, z=z, sigma=0.8)[0]}
            for m in MODES}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n", N_FRAMES)
def test_window_is_the_whole_call_bit_for_bit(case, vocoders, whole, mode, n):
    _, mels, olens, z, seeds = case
    v = vocoders[mode]
    for kind in KINDS:
        starts = _starts(kind, n)
        for noise, kw in (("seed", dict(seed=seeds)), ("z", dict(z=z))):
            if noise == "z" and kind in ("zero", "past"):
                continue
            audio, alens = v.window(mels, olens, torch.tensor(starts, device=DEV), n, sigma=0.8, **kw)
            assert audio.shape == (len(OLENS), n * HOP)
            assert alens.tolist() == [max(0, min(n, o - s)) * HOP for s, o in zip(starts, OLENS)]
            assert _same(audio, _expect(whole[mode][noise], OLENS, starts, n)), (mode, n, kind, noise)
    # reversed batch order, host starts, an int seed tensor reversed with it
    starts = _starts("interior", n)
    rev, _ = v.window(mels.flip(0).contiguous(), olens.flip(0).contiguous(), starts[::-1], n, sigma=0.8, seed=seeds.flip(0).contiguous())
    assert _same(rev.flip(0), _expect(whole[mode]["seed"], OLENS, starts, n)), (mode, n)


@pytest.mark.parametrize("mode", MODES)
def test_window_at_c256_and_each_utterance_alone(mode):
    from test_gpu_waveglow import make_oracle
    g = make_oracle(256, 2)
    v = _vocoder(g, mode)
    gen = torch.Generator().manual_seed(3)
    ol = [300, 40, 2]
    mels = (torch.randn(3, 300, 80, generator=gen) * 2 - 6).to(DEV)
    olens = torch.tensor(ol, device=DEV)
    full, _ = v(mels, olens, seed=7)
    n = 9
    for starts in ([0, 0, 0], [101, 35, 1], [200, 60, 0], [291, 31, 1]):
        audio, _ = v.window(mels, olens, starts, n, seed=7)
        assert _same(audio, _expect(full, ol, starts, n)), (mode, starts)
        for b in range(3):                                   # B = 1, its own Lmax, seed 7 + b
            one, _ = v.window(mels[b: b + 1, : ol[b]].contiguous(), olens[b: b + 1], starts[b], n, seed=7 + b)
            assert _same(one[0], audio[b]), (mode, starts, b)


def test_window_at_c512():
    from test_gpu_waveglow import make_oracle
    g = make_oracle(512, 3)
    v = _vocoder(g, "3xf16")
    gen = torch.Generator().manual_seed(4)
    ol = [230, 17]
    mels = (torch.randn(2, 230, 80, generator=gen) * 2 - 6).to(DEV)
    z = torch.randn(2, 8, 230 * STEPS, generator=gen).to(DEV)
    olens = torch.tensor(ol, device=DEV)
    full, _ = v(mels, olens, z=z)
    for starts, n in (([97, 3], 32), ([0, 0], 64), ([170, 16], 64)):
        audio, _ = v.window(mels, olens, starts, n, z=z)
        assert _same(audio, _expect(full, ol, starts, n)), (starts, n)


@pytest.mark.parametrize("mode", MODES)
def test_nan_outside_the_cone_changes_nothing(case, vocoders, whole, mode):
    _, mels, olens, z, seeds = case
    v = vocoders[mode]
    lo, hi = P.mel_reach()
    for kind, n in (("interior", 7), ("left", 32), ("end", 64), ("interior", 1)):
        starts = _starts(kind, n)
        nan_m, nan_z = mels.clone(), z.clone()
        for b, (s, o) in enumerate(zip(starts, OLENS)):
            keep = torch.zeros(mels.shape[1], dtype=torch.bool, device=DEV)
            keep[max(0, s - lo): min(o, s + n + hi)] = True
            nan_m[b, ~keep] = float("nan")
            keep_z = torch.zeros(z.shape[2], dtype=torch.bool, device=DEV)
            keep_z[max(0, s - P.halo()) * STEPS: min(o, s + n + P.halo()) * STEPS] = True
            nan_z[b, :, ~keep_z] = float("nan")
        audio, _ = v.window(nan_m, olens, starts, n, sigma=0.8, z=nan_z)          # raises on any status bit
        assert _same(audio, _expect(whole[mode]["z"], OLENS, starts, n)), (mode, kind, n)
        audio, _ = v.window(nan_m, olens, starts, n, sigma=0.8, seed=seeds)
        assert _same(audio, _expect(whole[mode]["seed"], OLENS, starts, n)), (mode, kind, n)


@pytest.mark.parametrize("mode", ["3xf16", "f16"])
def test_stream_concatenates_to_forward(case, vocoders, whole, mode):
    _, mels, olens, z, seeds = case
    v = vocoders[mode]
    for k in ((5, 32, 333) if mode == "3xf16" else (32,)):
        chunks = list(v.stream(mels, olens, chunk_frames=k, sigma=0.8, seed=seeds))
        assert len(chunks) == -(-max(OLENS) // k)
        assert _same(torch.cat([a for a, _ in chunks], 1), whole[mode]["seed"]), (mode, k)
        assert torch.equal(torch.stack([al for _, al in chunks]).sum(0), olens * HOP)
    chunks = list(v.stream(mels, olens, chunk_frames=64, sigma=0.8, z=z))
    assert _same(torch.cat([a for a, _ in chunks], 1), whole[mode]["z"])
    torch.manual_seed(21)                                    # seed=None: the whole call's one draw
    want, _ = v(mels, olens)
    torch.manual_seed(21)
    assert _same(torch.cat([a for a, _ in v.stream(mels, olens, chunk_frames=100)], 1), want)


@pytest.mark.parametrize("mode", MODES)
def test_chunked_forward_is_forward(case, vocoders, whole, mode):
    _, mels, olens, z, seeds = case
    v = vocoders[mode]
    for k in (7, 128, 2000):
        audio, alens = v(mels, olens, sigma=0.8, seed=seeds, chunk_frames=k)
        assert _same(audio, whole[mode]["seed"]) and torch.equal(alens, olens * HOP), (mode, k)
    audio, _ = v(mels, olens, sigma=0.8, z=z, chunk_frames=64)
    assert _same(audio, whole[mode]["z"])
    torch.manual_seed(5)
    want, _ = v(mels, olens)
    torch.manual_seed(5)
    assert _same(v(mels, olens, chunk_frames=50)[0], want), mode


def _raw_window(v, mels, olens, starts, n, seeds, audio, status, ws):
    dev = mels.device
    _lib.check(_lib.load().fs2_waveglow_window(v._handle(dev), _lib.ptr(mels), _lib.ptr(olens), _lib.ptr(starts), mels.shape[0],
                                               mels.shape[1], n, 0.8, _lib.ptr(seeds), None, _lib.ptr(audio), audio.shape[1],
                                               _lib.ptr(status), _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev)), "fs2_waveglow_window")


@pytest.mark.parametrize("mode", MODES)
def test_graph_replay_with_rewritten_starts_and_launch_count(case, vocoders, mode):
    _, mels, olens, _, seeds = case
    v = vocoders[mode]
    n = 13
    B = mels.shape[0]
    starts = torch.zeros(B, dtype=torch.int64, device=DEV)
    audio = torch.empty(B, n * HOP, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    ws = v._window_workspace(v._handle(mels.device), B, n, mels.device)
    lib = _lib.load()
    before = lib.fs2_kernel_launches()
    _raw_window(v, mels, olens, starts, n, seeds, audio, status, ws)
    assert lib.fs2_kernel_launches() - before == LAUNCHES[mode]
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):                 # the call allocates nothing and never synchronises
        _raw_window(v, mels, olens, starts, n, seeds, audio, status, ws)
    for kind in KINDS:
        st = _starts(kind, n)
        starts.copy_(torch.tensor(st))
        audio.fill_(7.0)
        graph.replay()
        torch.cuda.synchronize()
        assert int(status.item()) == 0
        eager, _ = v.window(mels, olens, st, n, sigma=0.8, seed=seeds)
        assert _same(audio, eager), (mode, kind)
    starts.copy_(torch.tensor([0, -1, 0, 0, 0, 0]))
    graph.replay()
    assert int(status.item()) == _lib.FS2_WAVEGLOW_BAD_START
    assert torch.all(audio[1] == 0) and not bool(torch.signbit(audio[1]).any())
    with pytest.raises(ValueError, match="starts"):
        v.window(mels, olens, starts, n, seed=seeds)


def test_range_is_raised_exactly_for_windows_whose_buffer_holds_the_spike(case, vocoders, whole):
    _, mels, olens, _, seeds = case
    f = 200                                                  # utterance 0 (420 frames)
    spiked = mels.clone()
    spiked[0, f] = 1e5                                       # an upsampling operand far above 4094
    n = 16
    for mode in ("3xf16", "f16"):
        v = vocoders[mode]
        with pytest.raises(ValueError, match="range"):
            v(spiked, olens, seed=seeds, sigma=0.8)
        for s in (f - 96 - n, f - 96 - n + 1, f, f + 96, f + 99, f + 100, 0, 400):
            starts = [s, 0, 0, 0, 0, 0]
            f0, f1, _, _ = P.buffer(s, n, OLENS[0])
            if f0 <= f + 3 and f < f1:                       # the buffer holds one of cond frames f .. f + 3
                with pytest.raises(ValueError, match="range"):
                    v.window(spiked, olens, starts, n, sigma=0.8, seed=seeds)
            else:
                # mel frame f lies outside the frames the window reads, so it is the unspiked whole call's audio
                audio, _ = v.window(spiked, olens, starts, n, sigma=0.8, seed=seeds)
                assert _same(audio, _expect(whole[mode]["seed"], OLENS, starts, n)), (mode, s)


def test_chunked_fp32_runs_what_the_whole_call_refuses():
    """B * Lmax * 32 above fp32's 65535 * 128 rows: the whole call refuses the batch, 1024-frame windows take it, and each
    utterance equals its own B = 1 whole call.  fp32's CUDA-core GEMMs compute every buffer row, so this is ~2e14 FLOP at
    C = 64 in a ~1.5 GB workspace."""
    from test_gpu_waveglow import make_oracle
    v = _vocoder(make_oracle(64, 6), "fp32")
    B, L = 8, 32770
    ol = [L, 3, 1100, 1, 40, 2049, 7, 500]
    gen = torch.Generator().manual_seed(8)
    mels = (torch.randn(B, L, 80, generator=gen) * 2 - 6).to(DEV)
    olens = torch.tensor(ol, device=DEV)
    with pytest.raises(ValueError, match="fp32"):
        v(mels, olens, seed=11)
    audio, _ = v(mels, olens, seed=11, chunk_frames=1024)
    for b in range(B):
        one, _ = v(mels[b: b + 1, : ol[b]].contiguous(), olens[b: b + 1], seed=11 + b)
        assert _same(audio[b, : ol[b] * HOP], one[0]), b
        assert torch.all(audio[b, ol[b] * HOP:] == 0)


def test_end_to_end_stream_after_synthesize():
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.hparams import load_hp
    model = FeedForwardTransformer(68, 80, load_hp())
    model.load_state_dict(synthetic_state_dict(0), strict=True)
    model = model.to(DEV).eval()
    fl = np.load(os.path.join(GOLDEN, "filelist64.npz"))
    with torch.no_grad():
        mels, olens, _ = model.synthesize(torch.from_numpy(fl["xs"][:16]).to(DEV), torch.from_numpy(fl["ilens"][:16]).to(DEV))
    torch.manual_seed(0)
    v = WaveGlowVocoder(n_channels=256).to(DEV)
    want, _ = v(mels, olens, sigma=0.6, seed=1)
    got = torch.cat([a for a, _ in v.stream(mels, olens, chunk_frames=32, sigma=0.6, seed=1)], 1)
    assert _same(got, want)
