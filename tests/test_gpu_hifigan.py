"""Batched HiFi-GAN vocoder on the H100 (HiFiGANVocoder, fs2_hifigan) against the oracle (oracle/hifigan_oracle.py) run
in float64 on the GPU, for V1 and V3 in every math mode: the audio, per-utterance bit-identity, the range check, graph
capture and the launch count, and the path from `synthesize`.

Weights: the oracle's default init with every g moved away from |v| (x U[0.5, 1.5)), then conv_post's g and bias scaled
so that the pre-tanh rms is 0.2 (tanh then hides no error); mels ~ N(-6, 2^2).  Gates are at most 3x the deviations
measured on an H100 (OBSERVED; DESIGN.md section 16).  The per-layer kernels are tested on their own in
test_gpu_hifigan_kernels.py."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from fastspeech2_b200 import _lib
from fastspeech2_b200.hifigan import CONFIGS, HOP, HiFiGANVocoder
from oracle import hifigan_oracle as O

pytestmark = pytest.mark.gpu
MODES = ["3xf16", "fp32", "f16", "tf32"]
CONFIG_NAMES = ["v1", "v3"]
# (max-abs, mean-abs) over the valid samples against the float64 oracle, measured on an H100 80GB HBM3 (700 W); the gates
# are 3x these
OBSERVED = {"v1": {"3xf16": (1.661e-6, 3.055e-7), "fp32": (3.577e-7, 5.890e-8), "f16": (1.282e-4, 2.142e-5), "tf32": (7.345e-4, 1.415e-4)},
            "v3": {"3xf16": (2.218e-6, 4.032e-7), "fp32": (5.107e-7, 8.145e-8), "f16": (3.875e-4, 5.008e-5), "tf32": (1.319e-3, 2.580e-4)}}
GATES = {c: {m: (3 * a, 3 * b) for m, (a, b) in o.items()} for c, o in OBSERVED.items()}
# 1 frame (the shortest utterance) and Lmax = 161: odd, so the stage rows Lmax * 8 are not a multiple of 16
OLENS = [37, 1, 160, 5, 64, 17, 161]


def test_fp32_class_gates_sit_below_the_f16_and_tf32_errors():
    for c in CONFIG_NAMES:
        for m in ("fp32", "3xf16"):
            for lossy in ("f16", "tf32"):
                assert GATES[c][m][0] < OBSERVED[c][lossy][0] and GATES[c][m][1] < OBSERVED[c][lossy][1], (c, m, lossy)


def _oracle(name, seed=0):
    torch.manual_seed(seed)
    g = O.Generator(CONFIGS[name])
    with torch.no_grad():
        for n, p in g.named_parameters():
            if n.endswith("weight_g"):
                p.mul_(torch.rand(p.shape) + 0.5)
    return g.eval()


def _calibrated(name, mels):
    """The oracle with conv_post scaled to a pre-tanh rms of 0.2 over the test utterances; -> (state dict, float64 audio,
    pre-tanh rms)."""
    g = _oracle(name)
    g64 = O.Generator(CONFIGS[name])
    g64.load_state_dict(g.state_dict())
    g64 = g64.eval().double().cuda()
    m64 = mels.double().cuda()
    n = int(sum(OLENS) * HOP)
    with torch.no_grad():
        rms = float(O.batched(g64, m64, OLENS, pre_tanh=True).pow(2).sum().div(n).sqrt())
        s = 0.2 / rms
        g64.conv_post.weight_g.mul_(s)
        g64.conv_post.bias.mul_(s)
        pre = O.batched(g64, m64, OLENS, pre_tanh=True)
        want = O.batched(g64, m64, OLENS).cpu()
    sd = {k: v.detach().float().cpu() for k, v in g64.state_dict().items()}
    return sd, want, float(pre.pow(2).sum().div(n).sqrt())


@pytest.fixture(scope="module")
def mels():
    gen = torch.Generator().manual_seed(1)
    return torch.randn(len(OLENS), max(OLENS), 80, generator=gen) * 2 - 6


@pytest.fixture(scope="module")
def cases(mels):
    out = {}
    for name in CONFIG_NAMES:
        sd, want, rms = _calibrated(name, mels)
        vocs = {}
        for m in MODES:
            v = HiFiGANVocoder(name, math_mode=m)
            v.load_state_dict(sd)
            vocs[m] = v.cuda().eval()
        out[name] = (sd, want, rms, vocs)
    return out


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", CONFIG_NAMES)
def test_audio_matches_oracle(cases, mels, name, mode):
    sd, want, rms, vocs = cases[name]
    assert 0.05 <= rms <= 0.5
    olens = torch.tensor(OLENS)
    audio, alens = vocs[mode](mels.cuda(), olens.cuda())
    audio = audio.cpu()
    assert audio.shape == (len(OLENS), max(OLENS) * HOP) and torch.equal(alens.cpu(), olens * HOP)
    err = (audio.double() - want).abs()
    mx, mean = float(err.max()), float(err.sum() / int(olens.sum() * HOP))
    print(f"\nhifigan {name} {mode}: max-abs {mx:.3e} mean-abs {mean:.3e} (pre-tanh rms {rms:.3f}, "
          f"audio rms {float(want.pow(2).sum().div(int(olens.sum() * HOP)).sqrt()):.3f})")
    gmax, gmean = GATES[name][mode]
    assert mx <= gmax, (name, mode, mx)
    assert mean <= gmean, (name, mode, mean)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", CONFIG_NAMES)
def test_per_utterance_bit_identity(cases, mels, name, mode):
    v = cases[name][3][mode]
    m, ol = mels.cuda(), torch.tensor(OLENS).cuda()
    audio, alens = v(m, ol)
    rev, _ = v(m.flip(0).contiguous(), ol.flip(0).contiguous())
    nan = m.clone()
    for b, n in enumerate(OLENS):
        nan[b, n:] = float("nan")                                 # frames past olens[b] are never read
    audio_nan, _ = v(nan, ol)
    assert torch.equal(audio_nan.view(torch.int32), audio.view(torch.int32)), mode
    B = len(OLENS)
    for b, n in enumerate(OLENS):
        one, l1 = v(m[b: b + 1, :n].contiguous(), ol[b: b + 1])
        assert int(l1[0]) == n * HOP == int(alens[b])
        assert torch.equal(audio[b, : n * HOP], one[0]), (mode, b)
        assert torch.equal(rev[B - 1 - b, : n * HOP], one[0]), (mode, b)
        assert torch.all(audio[b, n * HOP:].view(torch.int32) == 0), (mode, b)     # +0, no sign bit
    assert torch.isfinite(audio).all()


def test_bad_lengths_raise(cases, mels):
    v = cases["v3"][3]["3xf16"]
    for bad in ([0, 1, 2, 3, 4, 5, 6], [162, 1, 2, 3, 4, 5, 6]):
        with pytest.raises(ValueError, match="olens"):
            v(mels.cuda(), torch.tensor(bad).cuda())


def test_range_overflow_is_reported_not_clipped(cases, mels):
    sd = dict(cases["v3"][0])
    sd["conv_pre.weight_g"] = sd["conv_pre.weight_g"] * 3e4          # conv_pre's output far beyond 4094
    ol = torch.tensor(OLENS).cuda()
    for mode in ("f16", "3xf16"):
        v = HiFiGANVocoder("v3", math_mode=mode)
        v.load_state_dict(sd)
        with pytest.raises(ValueError, match="range"):
            v.cuda()(mels.cuda(), ol)
    v = HiFiGANVocoder("v3", math_mode="fp32")
    v.load_state_dict(sd)
    audio, _ = v.cuda()(mels.cuda(), ol)
    assert torch.isfinite(audio).all()


def _raw_call(v, mels, olens, audio, status, ws):
    dev = mels.device
    _lib.check(_lib.load().fs2_hifigan(v._handle(dev), _lib.ptr(mels), _lib.ptr(olens), mels.shape[0], mels.shape[1], _lib.ptr(audio),
                                       _lib.ptr(status), _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev)), "fs2_hifigan")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name,launches", [("v1", 160), ("v3", 49)])
def test_graph_capture_replays_bit_identically_and_launch_count(cases, mels, name, launches, mode):
    v = cases[name][3][mode]
    assert v.launches() == launches
    m, ol = mels.cuda().contiguous(), torch.tensor(OLENS).cuda()
    B, L = m.shape[:2]
    audio = torch.empty(B, L * HOP, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    ws = v._workspace(v._handle(m.device), B, L, m.device)
    lib = _lib.load()
    before = lib.fs2_kernel_launches()
    _raw_call(v, m, ol, audio, status, ws)
    assert lib.fs2_kernel_launches() - before == launches
    torch.cuda.synchronize()
    eager = audio.clone()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):                 # the call allocates nothing and never synchronises
        _raw_call(v, m, ol, audio, status, ws)
    audio.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    assert torch.equal(audio, eager)


def test_workspace_bytes_per_frame(cases):
    for name in CONFIG_NAMES:
        v = cases[name][3]["3xf16"]
        h = v._handle(torch.device("cuda", torch.cuda.current_device()))
        from fastspeech2_b200._kernel_module import query_bytes
        a, b = query_bytes("fs2_hifigan_workspace_bytes", h, 4, 1000), query_bytes("fs2_hifigan_workspace_bytes", h, 4, 2000)
        assert (b - a) / 4000 == 163840, (name, b - a)


def test_end_to_end_from_synthesize():
    """synthesize then the batched vocoder equals, per utterance, inference then a B = 1 vocoder call, bit for bit."""
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.hparams import load_hp
    model = FeedForwardTransformer(68, 80, load_hp())
    model.load_state_dict(synthetic_state_dict(0), strict=True)
    model = model.cuda().eval()
    fl = np.load(os.path.join(GOLDEN, "filelist64.npz"))
    xs, ilens = torch.from_numpy(fl["xs"][:6]).cuda(), torch.from_numpy(fl["ilens"][:6]).cuda()
    v = HiFiGANVocoder("v3").cuda()
    with torch.no_grad():
        mels, olens, _ = model.synthesize(xs, ilens)
        audio, alens = v(mels, olens)
        assert torch.equal(alens, olens * HOP)
        for b in range(xs.shape[0]):
            mel = model.inference(xs[b, : int(ilens[b])])
            one, _ = v(mel[None].contiguous(), torch.tensor([mel.shape[0]], device="cuda"))
            assert torch.equal(audio[b, : int(alens[b])], one[0]), b
            assert torch.all(audio[b, int(alens[b]):] == 0)
    assert torch.isfinite(audio).all() and float(audio.abs().max()) <= 1.0
