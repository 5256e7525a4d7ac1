"""Batched Griffin-Lim vocoder on the H100 (GriffinLimVocoder, fs2_griffin_lim) against the CPU oracle (oracle/gl_oracle.py):
mel inversion, audio after 0 and 2 iterations with given phases, convergence at 30 iterations, per-utterance independence
in every math mode, seeds, CUDA-graph capture, launch counts and the serving operator.

Tolerances, relative to the signal's peak: 3xf16 / fp32 2e-4 for the magnitudes and for the first inverse, 1e-3 after two
iterations (each pass re-derives the phase from the previous one, and near-zero bins have ill-conditioned phases).  f16 and
tf32 round every GEMM operand to 11 significant bits (relative 2^-11 ~ 4.9e-4 per operand, before a 1088-term sum and
three chained GEMMs): 5e-3 after 0 and 1.5e-2 after 2 iterations (measured on an H100: f16 5.3e-4 / 1.9e-3, tf32
1.4e-3 / 3.5e-3)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from fastspeech2_b200 import _lib
from fastspeech2_b200.vocoder import GriffinLimVocoder, mel_filterbank
from oracle import gl_oracle as G
from oracle import stft_oracle as O

pytestmark = pytest.mark.gpu
HOP, NFFT, CUT = 256, 1024, 513
MODES = ["3xf16", "fp32", "f16", "tf32"]


def _log_mels(olens, seed=0):
    """Log-mels of harmonic test signals (what TacotronSTFT.mel_spectrogram + log would give), [B, max(olens), 80]."""
    g = torch.Generator().manual_seed(seed)
    st = O.STFT(NFFT, HOP, NFFT)
    basis = torch.from_numpy(mel_filterbank(22050, NFFT, 80, 0.0, 8000.0))
    L = max(olens)
    out = torch.zeros(len(olens), L, 80)
    for b, n in enumerate(olens):
        t = torch.arange((n - 1) * HOP) / 22050.0
        f0 = 110.0 + 200.0 * float(torch.rand(1, generator=g))
        x = sum((0.3 / k) * torch.sin(2 * np.pi * k * f0 * t + float(torch.rand(1, generator=g)) * 6) for k in range(1, 6))
        x = x[None] + 0.003 * torch.randn(1, t.shape[0], generator=g)
        mag, _ = st.transform(x)
        out[b, :n] = torch.log(torch.clamp(basis @ mag[0, :, :n], min=1e-5)).T
    return out


def _peak_err(a, b):
    return float((a - b).abs().max()) / float(b.abs().max())


@pytest.fixture(scope="module")
def small():
    olens = [60, 45]
    mels = _log_mels(olens, 1)
    angles = (torch.rand(2, CUT, 60, generator=torch.Generator().manual_seed(2)) * 2 - 1) * np.pi
    return mels, torch.tensor(olens), angles


@pytest.mark.parametrize("mode", ["3xf16", "fp32"])
def test_mel_to_magnitude_vs_oracle(small, mode):
    mels, olens, _ = small
    v = GriffinLimVocoder(math_mode=mode).cuda()
    mag = v.mel_to_magnitude(mels.cuda(), olens.cuda()).cpu()
    P = G.mel_inverse(22050, NFFT, 80, 0.0, 8000.0)
    for b, n in enumerate(olens.tolist()):
        want = G.mel_to_magnitude(mels[b, :n], P)
        assert _peak_err(mag[b, :, :n], want) <= 2e-4, (mode, b)
        assert torch.all(mag[b, :, n:] == 0)


@pytest.mark.parametrize("mode,tol0,tol2", [("3xf16", 2e-4, 1e-3), ("fp32", 2e-4, 1e-3), ("f16", 5e-3, 1.5e-2), ("tf32", 5e-3, 1.5e-2)])
def test_audio_vs_oracle_with_given_angles(small, mode, tol0, tol2):
    mels, olens, angles = small
    v = GriffinLimVocoder(math_mode=mode).cuda()
    for n_iters, tol in ((0, tol0), (2, tol2)):
        audio, alens = v(mels.cuda(), olens.cuda(), n_iters=n_iters, angles=angles.cuda())
        want, want_lens = G.vocode(mels, olens, n_iters, angles)
        assert torch.equal(alens.cpu(), want_lens) and audio.shape == want.shape
        err = _peak_err(audio.cpu(), want)
        print(f"{mode} n_iters={n_iters}: max error / peak = {err:.2e}")
        assert err <= tol, (mode, n_iters, err)


def _spectral_convergence(y, M):
    mag, _ = O.STFT(NFFT, HOP, NFFT).transform(y)
    return float((mag - M).norm() / M.norm())


@pytest.mark.parametrize("momentum", [0.0, 0.99])
def test_convergence_at_30_iterations_like_the_oracle(small, momentum):
    mels, olens, angles = small
    n = int(olens[0])
    v = GriffinLimVocoder().cuda()
    audio, alens = v(mels[:1, :n].cuda(), olens[:1].cuda(), n_iters=30, momentum=momentum, angles=angles[:1, :, :n].cuda())
    P = G.mel_inverse(22050, NFFT, 80, 0.0, 8000.0)
    M = G.mel_to_magnitude(mels[0, :n], P)[None]
    want = G.griffin_lim(M, O.STFT(NFFT, HOP, NFFT), 30, angles[:1, :, :n], momentum)
    e_ours, e_ref = _spectral_convergence(audio.cpu(), M), _spectral_convergence(want, M)
    print(f"momentum {momentum}: spectral convergence {e_ours:.4f} (oracle {e_ref:.4f})")
    assert abs(e_ours - e_ref) <= 0.05 * e_ref, (e_ours, e_ref)


def test_fast_griffin_lim_converges_faster(small):
    mels, olens, _ = small
    v = GriffinLimVocoder().cuda()
    M = v.mel_to_magnitude(mels[:1].cuda(), olens[:1].cuda())[:, :, : int(olens[0])].cpu()
    sc = {}
    for momentum in (0.0, 0.99):
        audio, _ = v(mels[:1].cuda(), olens[:1].cuda(), n_iters=30, momentum=momentum, seed=5)
        sc[momentum] = _spectral_convergence(audio.cpu(), M)
    print("spectral convergence at 30 iterations:", sc)
    assert sc[0.99] < sc[0.0], sc


@pytest.fixture(scope="module")
def ragged():
    olens = np.load(os.path.join(GOLDEN, "filelist64.npz"))["olens"][:8].tolist()
    return _log_mels(olens, 3), torch.tensor(olens)


@pytest.mark.parametrize("mode", MODES)
def test_each_utterance_is_independent_of_its_batch(ragged, mode):
    mels, olens = ragged
    v = GriffinLimVocoder(math_mode=mode).cuda()
    m, ol = mels.cuda(), olens.cuda()
    seeds = torch.arange(8, dtype=torch.long, device="cuda") * 7919 + 1
    audio, alens = v(m, ol, n_iters=3, momentum=0.5, seed=seeds)
    poisoned = m.clone()
    for b, n in enumerate(olens.tolist()):
        poisoned[b, n:] = float("nan")
    audio_nan, _ = v(poisoned, ol, n_iters=3, momentum=0.5, seed=seeds)
    assert torch.equal(audio, audio_nan)
    for b, n in enumerate(olens.tolist()):
        a1, l1 = v(m[b: b + 1, :n], ol[b: b + 1], n_iters=3, momentum=0.5, seed=int(seeds[b]))
        assert int(alens[b]) == int(l1[0]) == (n - 1) * HOP
        assert torch.equal(audio[b, : (n - 1) * HOP], a1[0]), (mode, b)
        assert torch.all(audio[b, (n - 1) * HOP:] == 0), (mode, b)
    assert torch.isfinite(audio).all()


def test_seeds_reproduce_and_differ(small):
    mels, olens, _ = small
    v = GriffinLimVocoder().cuda()
    a, _ = v(mels.cuda(), olens.cuda(), n_iters=2, seed=11)
    b, _ = v(mels.cuda(), olens.cuda(), n_iters=2, seed=11)
    c, _ = v(mels.cuda(), olens.cuda(), n_iters=2, seed=12)
    assert torch.equal(a, b) and not torch.equal(a, c)


def test_lengths_too_short_for_reflect_padding_raise(small):
    mels, olens, _ = small
    v = GriffinLimVocoder().cuda()
    for bad in ([60, 2], [60, 61], [60, 0]):
        with pytest.raises(ValueError, match="olens"):
            v(mels.cuda(), torch.tensor(bad).cuda(), n_iters=1)
        with pytest.raises(ValueError, match="olens"):
            v.mel_to_magnitude(mels.cuda(), torch.tensor(bad).cuda())


def test_out_of_range_magnitudes_are_reported_not_clipped(small):
    mels, olens, _ = small
    v = GriffinLimVocoder().cuda()
    with pytest.raises(ValueError, match="range"):
        v(mels.cuda() + 12.0, olens.cuda(), n_iters=1)          # exp(mel) ~ e^12 exceeds the fp16 planes
    audio, _ = GriffinLimVocoder(math_mode="fp32").cuda()(mels.cuda() + 12.0, olens.cuda(), n_iters=1)
    assert torch.isfinite(audio).all()


def _raw_call(v, mels, olens, seeds, audio, status, ws):
    dev = mels.device
    _lib.check(_lib.load().fs2_griffin_lim(v._handle(dev), _lib.ptr(mels), _lib.ptr(olens), mels.shape[0], mels.shape[1], 4, 0.99,
                                           _lib.ptr(seeds), None, _lib.ptr(audio), _lib.ptr(status), _lib.ptr(ws), ws.numel(),
                                           _lib.stream_ptr(dev)), "fs2_griffin_lim")


def test_graph_capture_replays_bit_identically(ragged):
    mels, olens = ragged
    v = GriffinLimVocoder().cuda()
    m, ol = mels[:4].cuda().contiguous(), olens[:4].cuda()
    L = m.shape[1]
    seeds = torch.tensor([1, 2, 3, 4], device="cuda")
    audio = torch.empty(4, (L - 1) * HOP, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    ws = v._workspace(v._handle(m.device), 4, L, m.device)
    _raw_call(v, m, ol, seeds, audio, status, ws)
    torch.cuda.synchronize()
    eager = audio.clone()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):                 # the call allocates nothing and never synchronises
        _raw_call(v, m, ol, seeds, audio, status, ws)
    audio.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    assert torch.equal(audio, eager)


def test_kernel_launches_are_linear_in_iterations(small):
    mels, olens, _ = small
    v = GriffinLimVocoder().cuda()
    lib = _lib.load()
    v(mels.cuda(), olens.cuda(), n_iters=1)
    counts = {}
    for n in (0, 1, 2, 5):
        before = lib.fs2_kernel_launches()
        v(mels.cuda(), olens.cuda(), n_iters=n)
        counts[n] = lib.fs2_kernel_launches() - before
    b = counts[1] - counts[0]
    assert b == 4 and all(counts[n] == counts[0] + b * n for n in counts), counts
    assert counts[0] == 5, counts


def test_serving_operator_matches_eager_synthesize_plus_vocoder():
    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.hparams import load_hp
    from fastspeech2_b200.serving import scripted
    model = FeedForwardTransformer(68, 80, load_hp())
    model.load_state_dict(synthetic_state_dict(0), strict=True)
    model = model.cuda().eval()
    fl = np.load(os.path.join(GOLDEN, "filelist64.npz"))
    rows = [2, 0, 5]                                              # ragged real phoneme sequences
    xs = torch.from_numpy(fl["xs"][rows]).cuda()
    ilens = torch.from_numpy(fl["ilens"][rows]).cuda()
    xs = xs[:, : int(ilens.max())].contiguous()
    one = torch.ones((), device="cuda")
    speed = torch.tensor([1.0, 1.2, 0.9], device="cuda")
    with torch.no_grad():
        mels, olens, _ = model.synthesize(xs, ilens, speed=speed)
        want, want_lens = GriffinLimVocoder.from_hp(load_hp(), math_mode=model.precision).cuda()(mels, olens, n_iters=5, momentum=0.99, seed=9)
    served = scripted(model)
    audio, alens = served.synthesize_audio(xs, ilens, speed, one, one, 5, 0.99, 9)
    assert torch.equal(alens, want_lens) and torch.equal(audio, want)
