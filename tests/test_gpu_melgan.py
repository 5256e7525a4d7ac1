"""Batched MelGAN vocoder on the H100 (MelGANVocoder, fs2_melgan) against the oracle (oracle/melgan_oracle.py) run in
float64 on the GPU: audio in every math mode, per-utterance bit-identity, `inference`, the range check, graph capture and launch count, the
drop-in hub hook and the path from `synthesize`.

Weights: the oracle's default init with every g moved away from |v| (x U[0.5, 1.5)); mels ~ N(-6, 2^2).  Gates on the
audio (output rms ~0.1) are a small multiple of the measured deviations (see GATES; DESIGN.md section 8).  The
per-layer kernels are tested on their own in test_gpu_melgan_kernels.py."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from fastspeech2_b200 import _lib
from fastspeech2_b200 import dropin_run
from fastspeech2_b200.melgan import HOP, MelGANVocoder
from oracle import melgan_oracle as O

pytestmark = pytest.mark.gpu
MODES = ["3xf16", "fp32", "f16", "tf32"]
# (max-abs, mean-abs) over the valid samples against the float64 oracle; measured on an H100: 3xf16 2.1e-7 / 3.7e-8,
# fp32 1.9e-7 / 3.2e-8, f16 7.3e-5 / 1.4e-5, tf32 1.6e-4 / 9.7e-5.  The fp32-class gates sit far below the f16 / tf32
# errors, so a mode that silently lost its lo planes or fell back to tf32 fails them.
GATES = {"3xf16": (1e-6, 2e-7), "fp32": (1e-6, 2e-7), "f16": (3e-4, 6e-5), "tf32": (6e-4, 4e-4)}
# 1 frame (the shortest utterance), 900 frames, and Lmax = 901: Lmax + 10 odd, so stage 1 has (Lmax + 10) * 8 rows per
# utterance, not a multiple of 16
OLENS = [37, 1, 900, 5, 260, 64, 901]


def _oracle(seed=0):
    torch.manual_seed(seed)
    g = O.Generator()
    with torch.no_grad():
        for name, p in g.named_parameters():
            if name.endswith("weight_g"):
                p.mul_(torch.rand(p.shape) + 0.5)
    return g.eval()


@pytest.fixture(scope="module")
def case():
    g = _oracle(0)
    gen = torch.Generator().manual_seed(1)
    L = max(OLENS)
    mels = torch.randn(len(OLENS), L, 80, generator=gen) * 2 - 6
    olens = torch.tensor(OLENS)
    g64 = O.Generator()
    g64.load_state_dict(g.state_dict())
    g64 = g64.eval().double().cuda()
    with torch.no_grad():
        want = O.batched(g64, mels.double().cuda(), OLENS).cpu()
    del g64
    return g, mels, olens, want


@pytest.fixture(scope="module")
def vocoders(case):
    g = case[0]
    out = {}
    for m in MODES:
        v = MelGANVocoder(math_mode=m)
        v.load_state_dict(g.state_dict())
        out[m] = v.cuda().eval()
    return out


@pytest.mark.parametrize("mode", MODES)
def test_audio_matches_oracle(case, vocoders, mode):
    g, mels, olens, want = case
    audio, alens = vocoders[mode](mels.cuda(), olens.cuda())
    audio = audio.cpu()
    assert audio.shape == (len(OLENS), max(OLENS) * HOP) and torch.equal(alens.cpu(), olens * HOP)
    err = (audio.double() - want).abs()
    mx, mean = float(err.max()), float(err.sum() / int(olens.sum() * HOP))
    print(f"\nmelgan {mode}: max-abs {mx:.3e} mean-abs {mean:.3e} (audio rms {float(want.pow(2).mean().sqrt()):.3f})")
    gmax, gmean = GATES[mode]
    assert mx <= gmax, (mode, mx)
    assert mean <= gmean, (mode, mean)


@pytest.mark.parametrize("mode", MODES)
def test_per_utterance_bit_identity(case, vocoders, mode):
    _, mels, olens, _ = case
    v = vocoders[mode]
    m, ol = mels.cuda(), olens.cuda()
    audio, alens = v(m, ol)
    rev, _ = v(m.flip(0).contiguous(), ol.flip(0).contiguous())
    nan = m.clone()
    for b, n in enumerate(OLENS):
        nan[b, n:] = float("nan")                                 # frames past olens[b] are never read
    audio_nan, _ = v(nan, ol)
    assert torch.equal(audio_nan, audio), mode
    B = len(OLENS)
    for b, n in enumerate(OLENS):
        one, l1 = v(m[b: b + 1, :n].contiguous(), ol[b: b + 1])
        assert int(l1[0]) == n * HOP == int(alens[b])
        assert torch.equal(audio[b, : n * HOP], one[0]), (mode, b)
        assert torch.equal(rev[B - 1 - b, : n * HOP], one[0]), (mode, b)
        assert torch.all(audio[b, n * HOP:] == 0), (mode, b)
    assert torch.isfinite(audio).all()


@pytest.mark.parametrize("mode", MODES)
def test_inference_is_the_quantised_batched_audio(case, vocoders, mode):
    g, mels, olens, _ = case
    v = vocoders[mode]
    b = 4
    n = OLENS[b]
    mel = mels[b, :n].T[None].contiguous()                       # [1, 80, T], as inference.py passes it
    i16 = v.inference(mel.cuda())
    assert i16.dtype == torch.int16 and i16.shape == (n * HOP,)
    audio, _ = v(mels.cuda(), olens.cuda())
    assert torch.equal(i16, MelGANVocoder.quantize(audio[b, : n * HOP]))
    if mode in ("fp32", "3xf16"):
        with torch.no_grad():
            want = g.inference(mel)
        assert int((i16.cpu().int() - want.int()).abs().max()) <= 1


def test_range_overflow_is_reported_not_clipped(case):
    g, mels, olens, _ = case
    sd = dict(g.state_dict())
    sd["generator.1.weight_g"] = sd["generator.1.weight_g"] * 3e4          # first conv's output far beyond 4094
    for mode in ("f16", "3xf16"):
        v = MelGANVocoder(math_mode=mode)
        v.load_state_dict(sd)
        with pytest.raises(ValueError, match="range"):
            v.cuda()(mels.cuda(), olens.cuda())
    v = MelGANVocoder(math_mode="fp32")
    v.load_state_dict(sd)
    audio, _ = v.cuda()(mels.cuda(), olens.cuda())
    assert torch.isfinite(audio).all()


def test_bad_lengths_raise(case, vocoders):
    _, mels, _, _ = case
    for bad in ([0, 1, 2, 3, 4, 5, 6], [902, 1, 2, 3, 4, 5, 6]):
        with pytest.raises(ValueError, match="olens"):
            vocoders["3xf16"](mels.cuda(), torch.tensor(bad).cuda())


def _raw_call(v, mels, olens, audio, status, ws):
    dev = mels.device
    _lib.check(_lib.load().fs2_melgan(v._handle(dev), _lib.ptr(mels), _lib.ptr(olens), mels.shape[0], mels.shape[1], _lib.ptr(audio),
                                      _lib.ptr(status), _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev)), "fs2_melgan")


# 3 + 4 * 2 + 12 per unfused and 3 per fused ResStack + 1: f16 fuses the stages with C <= 128, 3xf16 those with C <= 64
@pytest.mark.parametrize("mode,launches", [("3xf16", 3 + 8 + 2 * 12 + 2 * 3 + 1), ("f16", 3 + 8 + 12 + 3 * 3 + 1),
                                            ("tf32", 3 + 8 + 4 * 12 + 1), ("fp32", 60)])
def test_graph_capture_replays_bit_identically_and_launch_count(case, vocoders, mode, launches):
    _, mels, olens, _ = case
    v = vocoders[mode]
    m, ol = mels[:, :300].cuda().contiguous(), olens.clamp(max=300).cuda()
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


def test_dropin_hub_checkpoint_matches_oracle(case, tmp_path, monkeypatch):
    g, mels, _, _ = case
    path = tmp_path / "melgan.pt"
    torch.save({"model_g": g.state_dict(), "model_d": {}, "step": 0, "epoch": 0}, path)
    monkeypatch.setattr(torch.hub, "load", lambda *a, **k: pytest.fail("the network hub must not be reached"))
    dropin_run.install_melgan_hub(str(path))
    vocoder = torch.hub.load("seungwonpark/melgan", "melgan")
    vocoder.eval(inference=False)
    vocoder.cuda()
    mel = mels[0, :37].T[None].contiguous()
    with torch.no_grad():
        got = vocoder.inference(mel.cuda()).cpu()
        want = g.inference(mel)
    assert got.shape == want.shape and int((got.int() - want.int()).abs().max()) <= 1


def test_end_to_end_from_synthesize():
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.hparams import load_hp
    model = FeedForwardTransformer(68, 80, load_hp())
    model.load_state_dict(synthetic_state_dict(0), strict=True)
    model = model.cuda().eval()
    fl = np.load(os.path.join(GOLDEN, "filelist64.npz"))
    with torch.no_grad():
        mels, olens, _ = model.synthesize(torch.from_numpy(fl["xs"]).cuda(), torch.from_numpy(fl["ilens"]).cuda())
    v = MelGANVocoder().cuda()
    audio, alens = v(mels, olens)
    B, L = mels.shape[:2]
    assert audio.shape == (B, L * HOP) and audio.dtype == torch.float32
    assert torch.equal(alens, olens * HOP)
    assert torch.isfinite(audio).all() and float(audio.abs().max()) <= 1.0
    for b in range(B):
        assert torch.all(audio[b, int(alens[b]):] == 0)
