"""Batched iSTFTNet vocoder on the H100 (ISTFTNetVocoder, fs2_istftnet) against the oracle (oracle/istftnet_oracle.py) run
in float64 on the GPU, in every math mode: the audio, the head alone (fs2_op_istftnet_head) against the float64 index
form, per-utterance bit-identity, graph capture and the launch count, the workspace and the path from `synthesize`.

Weights: the oracle's default init with every g moved away from |v| (x U[0.5, 1.5)), then conv_post's g scaled and the
magnitude biases set so that the log-magnitudes lie in [-8, 2], where a trained model puts them, rather than where exp()
explodes; mels ~ N(-6, 2^2).  Errors are relative: max-abs over max |audio|.  Gates are 3x the errors measured on an H100
(OBSERVED; DESIGN.md section 19)."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from fastspeech2_b200 import _lib
from fastspeech2_b200._kernel_module import query_bytes
from fastspeech2_b200.istftnet import CONFIGS, HOP, ISTFTNetVocoder
from oracle import istftnet_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _istftnet_head as H  # noqa: E402

pytestmark = pytest.mark.gpu
MODES = ["3xf16", "fp32", "f16", "tf32"]
# max-abs error over max |audio| against the float64 oracle, measured on an H100 80GB HBM3 (700 W); the gates are 3x these
OBSERVED = {"3xf16": 3.219e-5, "fp32": 2.751e-6, "f16": 9.519e-4, "tf32": 9.153e-3}
GATES = {m: 3 * e for m, e in OBSERVED.items()}
OBSERVED_HEAD = 6.759e-6      # fs2_op_istftnet_head against the float64 index form, same measure, worst of the three C
OLENS = [37, 1, 160, 5, 64, 17, 161]


def _calibrated_oracle(mels, olens, seed=0):
    """The float64 oracle with perturbed g and conv_post set so that y[:9] lies in [-8, 2] on these utterances."""
    torch.manual_seed(seed)
    g = O.Generator(CONFIGS["v1"])
    with torch.no_grad():
        for n, p in g.named_parameters():
            if n.endswith("weight_g"):
                p.mul_(torch.rand(p.shape) + 0.5)
    g = g.double().eval()
    M = g.n_fft // 2 + 1
    with torch.no_grad():
        y = O.batched(g, mels.double(), olens, pre_head=True)
        z = torch.cat([y[b, :, : n * 64 + 1] for b, n in enumerate(olens)], 1) - g.conv_post.bias[:, None]
        s = 5.0 / float(z.abs().max())
        g.conv_post.weight_g.mul_(s)
        g.conv_post.bias.mul_(s)
        g.conv_post.bias[:M] = -3.0
        y = O.batched(g, mels.double(), olens, pre_head=True)
        ym = torch.cat([y[b, :M, : n * 64 + 1] for b, n in enumerate(olens)], 1)
    assert -8.0 - 1e-9 <= float(ym.min()) and float(ym.max()) <= 2.0 + 1e-9
    return g


@pytest.fixture(scope="module")
def mels():
    gen = torch.Generator().manual_seed(1)
    return torch.randn(len(OLENS), max(OLENS), 80, generator=gen) * 2 - 6


@pytest.fixture(scope="module")
def case(mels):
    g = _calibrated_oracle(mels, OLENS)
    gc = g.cuda()
    with torch.no_grad():
        want = O.batched(gc, mels.double().cuda(), OLENS).cpu()
    sd = {k: v.detach().float().cpu() for k, v in g.state_dict().items()}
    vocs = {}
    for m in MODES:
        v = ISTFTNetVocoder("v1", math_mode=m)
        v.load_state_dict(sd)
        vocs[m] = v.cuda().eval()
    return sd, want, vocs


@pytest.mark.parametrize("mode", MODES)
def test_audio_matches_oracle(case, mels, mode):
    sd, want, vocs = case
    olens = torch.tensor(OLENS)
    audio, alens = vocs[mode](mels.cuda(), olens.cuda())
    audio = audio.cpu()
    assert audio.shape == (len(OLENS), max(OLENS) * HOP) and torch.equal(alens.cpu(), olens * HOP)
    rel = float((audio.double() - want).abs().max() / want.abs().max())
    print(f"\nistftnet v1 {mode}: max-abs / max |audio| {rel:.3e} (max |audio| {float(want.abs().max()):.3e})")
    assert rel <= GATES[mode], (mode, rel)


@pytest.mark.parametrize("C", [32, 128, 512])
def test_head_op_matches_the_float64_index_form(C):
    """fs2_op_istftnet_head on utterances of 1, 2 and all Lp rows against tests/_istftnet_head.py in float64."""
    B, Lp, N, hop = 3, 700, 16, 4
    gen = torch.Generator().manual_seed(C)
    x = torch.randn(B, Lp, C, generator=gen)
    w = torch.randn(N + 2, C, 7, generator=gen) / (7 * C) ** 0.5
    b = torch.randn(N + 2, generator=gen) * 0.5
    b[: N // 2 + 1] -= 3.0
    lens = [1, 2, Lp]
    audio = torch.empty(B, Lp * hop, device="cuda")
    xd, wd, bd = x.cuda().contiguous(), w.cuda().contiguous(), b.cuda().contiguous()
    ld = torch.tensor(lens, device="cuda")
    _lib.check(_lib.load().fs2_op_istftnet_head(C, N, hop, _lib.ptr(xd), _lib.ptr(ld), B, Lp, _lib.ptr(wd), _lib.ptr(bd), _lib.ptr(audio),
                                                _lib.stream_ptr(xd.device)), "fs2_op_istftnet_head")
    audio = audio.cpu()
    worst = 0.0
    for i, n in enumerate(lens):
        want = H.head(x[i, :n].double().numpy(), w.double().numpy(), b.double().numpy(), N, hop)
        got = audio[i, : n * hop].double().numpy()
        worst = max(worst, float(np.abs(got - want).max() / np.abs(want).max()))
        assert torch.all(audio[i, n * hop:].view(torch.int32) == 0), (C, n)
    print(f"\nistftnet head C={C}: max-abs / max |audio| {worst:.3e}")
    assert worst <= 3 * OBSERVED_HEAD, (C, worst)


@pytest.mark.parametrize("mode", MODES)
def test_per_utterance_bit_identity(case, mels, mode):
    v = case[2][mode]
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


def test_bad_lengths_raise(case, mels):
    v = case[2]["3xf16"]
    for bad in ([0, 1, 2, 3, 4, 5, 6], [162, 1, 2, 3, 4, 5, 6]):
        with pytest.raises(ValueError, match="olens"):
            v(mels.cuda(), torch.tensor(bad).cuda())


def _raw_call(v, mels, olens, audio, status, ws):
    dev = mels.device
    _lib.check(_lib.load().fs2_istftnet(v._handle(dev), _lib.ptr(mels), _lib.ptr(olens), mels.shape[0], mels.shape[1], _lib.ptr(audio),
                                        _lib.ptr(status), _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev)), "fs2_istftnet")


@pytest.mark.parametrize("mode", MODES)
def test_graph_capture_replays_bit_identically_and_launch_count(case, mels, mode):
    v = case[2][mode]
    assert v.launches() == 82
    m, ol = mels.cuda().contiguous(), torch.tensor(OLENS).cuda()
    B, L = m.shape[:2]
    audio = torch.empty(B, L * HOP, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    ws = v._workspace(v._handle(m.device), B, L, m.device)
    lib = _lib.load()
    before = lib.fs2_kernel_launches()
    _raw_call(v, m, ol, audio, status, ws)
    assert lib.fs2_kernel_launches() - before == 82
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


def test_workspace_bytes_per_frame(case):
    """Five buffers of max_s up_s C_s = 64 * 128 floats per frame, as HiFi-GAN V1's 256 * 32."""
    v = case[2]["3xf16"]
    h = v._handle(torch.device("cuda", torch.cuda.current_device()))
    a, b = query_bytes("fs2_istftnet_workspace_bytes", h, 4, 1000), query_bytes("fs2_istftnet_workspace_bytes", h, 4, 2000)
    assert (b - a) / 4000 == 163840


def test_end_to_end_from_synthesize():
    """synthesize then the batched vocoder equals, per utterance, inference then a B = 1 vocoder call, bit for bit."""
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.hparams import load_hp
    model = FeedForwardTransformer(68, 80, load_hp())
    model.load_state_dict(synthetic_state_dict(0), strict=True)
    model = model.cuda().eval()
    fl = np.load(os.path.join(GOLDEN, "filelist64.npz"))
    xs, ilens = torch.from_numpy(fl["xs"][:6]).cuda(), torch.from_numpy(fl["ilens"][:6]).cuda()
    torch.manual_seed(0)
    v = ISTFTNetVocoder("v1").cuda()
    with torch.no_grad():
        mels, olens, _ = model.synthesize(xs, ilens)
        audio, alens = v(mels, olens)
        assert torch.equal(alens, olens * HOP)
        for b in range(xs.shape[0]):
            mel = model.inference(xs[b, : int(ilens[b])])
            one, _ = v(mel[None].contiguous(), torch.tensor([mel.shape[0]], device="cuda"))
            assert torch.equal(audio[b, : int(alens[b])], one[0]), b
            assert torch.all(audio[b, int(alens[b]):] == 0)
    assert torch.isfinite(audio).all()
