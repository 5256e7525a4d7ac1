"""Batched WaveGlow vocoder on the H100 (WaveGlowVocoder, fs2_waveglow) and the dilated tap GEMM under it
(fs2_op_tap_gemm_dil), against float64: the dilated GEMM in all four families, audio in every math mode against the
oracle (oracle/waveglow_oracle.py) with the same z, the round trip through the oracle's forward direction, sigma = 0,
per-utterance bit-identity, the noise, the range check, graph capture and launch count, the drop-in hub hook and the path
from `synthesize`.

Weights: the oracle's init with every g moved away from |v| (x U[0.5, 1.5)) and `end` drawn as N(0, 1 / C), bias
N(0, 0.1^2), so that the couplings are far from the identity (mean |log s| ~ 0.3, up to ~1); mels ~ N(-6, 2^2).  Gates on the audio
are a small multiple of the deviations measured on an H100 (GATES; DESIGN.md section 9)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN
from fastspeech2_b200 import _lib
from fastspeech2_b200 import dropin_run
from fastspeech2_b200.waveglow import HOP, STEPS, WaveGlowVocoder
from oracle import waveglow_oracle as O
from test_gpu_tap_gemm import MODE, Guarded, bits, f16_operands, to_tf32, TF32_CONVERSION

pytestmark = pytest.mark.gpu
DEV = "cuda"
MODES = ["3xf16", "fp32", "f16", "tf32"]
OLENS = [37, 1, 64, 5, 2]
# (max-abs, mean-abs) over the valid samples, as fractions of the oracle's max |audio| (A = 879 in the C = 256 case: these
# weights make a loud, ill-conditioned model, where the eager fp32 oracle itself is 12.4 / 6.3e-3 off float64).  Measured
# on an H100, in units of A (DESIGN.md section 9):
#   C = 256: 3xf16 1.0e-4 / 7.4e-8, fp32 1.4e-5 / 7.2e-9, f16 7.5e-3 / 5.7e-6, tf32 0.19 / 4.8e-5;
#   C = 512, 3xf16: 4.4e-5 / 4.6e-7 (A = 121); sigma = 0, 3xf16: 7.0e-6 / 1.0e-6 (A = 2.5);
#   C = 64: 3xf16 1.6e-5 / 1.3e-7, f16 4.6e-3 / 3.3e-5 (A = 109).
# The fp32-class gates sit below the f16 / tf32 errors, so a mode that silently lost its lo planes or fell back to tf32
# fails them.
GATES = {"3xf16": (5e-4, 2e-6), "fp32": (5e-4, 2e-6), "f16": (3e-2, 1e-4), "tf32": (0.5, 2e-4)}


# ---- the dilated tap GEMM ------------------------------------------------------------------------------------------
def dil_gemm(fam, x, w, bias, lens, dil):
    """One fs2_op_tap_gemm_dil call on a sentinel-guarded output [B, L, N]."""
    lib = _lib.load()
    B, L, K = x.shape
    taps, N, _ = w.shape
    g = Guarded(B * L * N, torch.float32)
    rc = lib.fs2_op_tap_gemm_dil(MODE[fam], _lib.ptr(x), B, L, K, _lib.ptr(w), _lib.ptr(bias), N, taps, 0, None, _lib.ptr(lens),
                                 _lib.ptr(g.view), None, 0, 0, None, 0, dil, _lib.stream_ptr(x.device))
    _lib.check(rc, "fs2_op_tap_gemm_dil")
    torch.cuda.synchronize()
    assert g.intact(), f"{fam}: a store landed outside the output"
    return g.view.view(B, L, N)


def dil_reference(x, w, bias, lens, dil):
    """float64 nn.Conv1d(dilation = dil, padding = pad * dil) per utterance, as shifted matmuls; zeros past lens."""
    taps, L = w.shape[0], x.shape[1]
    pad = (taps - 1) // 2 * dil
    xp = F.pad(x.double(), (0, 0, pad, pad))
    y = sum(xp[:, j * dil: j * dil + L] @ w[j].double().T for j in range(taps)) + bias.double()
    return y.masked_fill(~(torch.arange(L, device=x.device)[None, :] < lens[:, None])[..., None], 0.0)


def dil_gates(fam, x, w):
    if fam == "fp32":
        return [("exact", x, w, 2e-5, 2e-6)]
    if fam == "3xf16":
        return [("exact", x, w, 2e-4, 2e-5)]
    if fam == "f16":
        return [("fp16 operands", *f16_operands(x, w), 5e-4, 5e-5), ("exact", x, w, 1e-2, 1e-3)]
    return [("tf32 operands", to_tf32(x, TF32_CONVERSION), to_tf32(w, TF32_CONVERSION), 5e-4, 5e-5), ("exact", x, w, 1e-2, 1e-3)]


@pytest.mark.parametrize("dil", [1, 2, 4, 8, 16, 32, 64, 128])
@pytest.mark.parametrize("fam", ["fp32", "tf32", "f16", "3xf16"])
def test_dilated_tap_gemm_matches_float64(fam, dil):
    """Ragged batch: a 300-row utterance (three tiles), a 32-row one (one step frame, shorter than dilations 64 and 128),
    a 77-row one (a packed tail) and an empty one; the input is zero past lens, as the contract asks."""
    gen = torch.Generator().manual_seed(dil)
    B, L, K, N, taps = 4, 300, 64, 128, 3
    lens = torch.tensor([300, 32, 77, 0], device=DEV)
    x = torch.randn(B, L, K, generator=gen).to(DEV)
    x = x.masked_fill(~(torch.arange(L, device=DEV)[None, :] < lens[:, None])[..., None], 0.0).contiguous()
    w = (torch.randn(taps, N, K, generator=gen) / (K * taps) ** 0.5).to(DEV).contiguous()
    bias = (torch.randn(N, generator=gen) * 0.1).to(DEV)
    got = dil_gemm(fam, x, w, bias, lens, dil)
    mask = torch.arange(L, device=DEV)[None, :] < lens[:, None]
    assert bool((got[~mask] == 0).all()) and not bool(torch.signbit(got[~mask]).any()), "rows past lens must be +0"
    for label, xx, ww, gmax, gmean in dil_gates(fam, x, w):
        err = (got.double() - dil_reference(xx, ww, bias, lens, dil))[mask].abs()
        print(f"GATE {fam:6s} dil {dil:3d} {label:14s} max {float(err.max()):.3e} / {gmax:.0e}  mean {float(err.mean()):.3e} / {gmean:.0e}")
        assert float(err.max()) <= gmax and float(err.mean()) <= gmean, (fam, dil, label)


def test_dilation_one_is_the_undilated_call():
    gen = torch.Generator().manual_seed(7)
    x = torch.randn(2, 150, 64, generator=gen).to(DEV)
    w = torch.randn(3, 64, 64, generator=gen).to(DEV) / 14
    bias = torch.zeros(64, device=DEV)
    lens = torch.tensor([150, 150], device=DEV)
    lib = _lib.load()
    for fam in MODE:
        a = dil_gemm(fam, x, w, bias, lens, 1)
        b = torch.empty_like(a)
        _lib.check(lib.fs2_op_tap_gemm_ex(MODE[fam], _lib.ptr(x), 2, 150, 64, _lib.ptr(w), _lib.ptr(bias), 64, 3, 0, None, _lib.ptr(lens),
                                          _lib.ptr(b), None, 0, 0, None, 0, _lib.stream_ptr(x.device)), "fs2_op_tap_gemm_ex")
        torch.cuda.synchronize()
        assert torch.equal(bits(a), bits(b)), fam
    assert lib.fs2_op_tap_gemm_dil(MODE["fp32"], _lib.ptr(x), 2, 150, 64, _lib.ptr(w), None, 64, 3, 0, None, None, _lib.ptr(a), None,
                                   0, 0, None, 0, 0, _lib.stream_ptr(x.device)) == -1


# ---- the vocoder ---------------------------------------------------------------------------------------------------
def make_oracle(C, seed=0):
    torch.manual_seed(seed)
    g = O.WaveGlow(C)
    with torch.no_grad():
        for name, p in g.named_parameters():
            if name.endswith("weight_g"):
                p.mul_(torch.rand(p.shape) + 0.5)
        for wn in g.WN:
            wn.end.weight.normal_(0, 1.0 / C ** 0.5)
            wn.end.bias.normal_(0, 0.1)
    return g.eval()


def clone(g):
    c = O.WaveGlow(g.WN[0].n_channels)                 # deepcopy does not take weight-normed modules
    c.load_state_dict(g.state_dict())
    return c.eval()


def vocoder(g, mode):
    v = WaveGlowVocoder(n_channels=g.WN[0].n_channels, math_mode=mode)
    v.load_state_dict(g.state_dict())
    return v.to(DEV).eval()


@pytest.fixture(scope="module")
def case():
    g = make_oracle(256, 0)
    gen = torch.Generator().manual_seed(1)
    B, L = len(OLENS), max(OLENS)
    mels = torch.randn(B, L, 80, generator=gen) * 2 - 6
    z = torch.randn(B, 8, L * STEPS, generator=gen)
    olens = torch.tensor(OLENS)
    g64 = clone(g).double().to(DEV)
    with torch.no_grad():
        want = O.batched(g64, mels.double().to(DEV), OLENS, z.double().to(DEV)).float().cpu()
    return g, g64, mels, olens, z, want


@pytest.fixture(scope="module")
def vocoders(case):
    return {m: vocoder(case[0], m) for m in MODES}


def audio_error(got, want, olens):
    valid = torch.arange(want.shape[1])[None, :] < (olens * HOP)[:, None]
    err = (got.double() - want.double()).abs()[valid]
    return float(err.max()), float(err.mean())


def check_gate(mode, got, want, olens, label):
    A = float(want.abs().max())
    mx, mean = audio_error(got, want, olens)
    gmax, gmean = GATES[mode]
    print(f"\nwaveglow {label} {mode}: max-abs {mx:.3e} ({mx / A:.2e} A) mean-abs {mean:.3e} ({mean / A:.2e} A), A = {A:.3g}")
    assert mx <= gmax * A and mean <= gmean * A, (mode, label, mx / A, mean / A)


@pytest.mark.parametrize("mode", MODES)
def test_audio_matches_oracle(case, vocoders, mode):
    g, _, mels, olens, z, want = case
    audio, alens = vocoders[mode](mels.to(DEV), olens.to(DEV), z=z.to(DEV))
    audio = audio.cpu()
    assert audio.shape == (len(OLENS), max(OLENS) * HOP) and torch.equal(alens.cpu(), olens * HOP)
    check_gate(mode, audio, want, olens, "C=256")


def test_audio_matches_oracle_c512():
    g = make_oracle(512, 3)
    gen = torch.Generator().manual_seed(4)
    ol = [9, 2]
    mels = torch.randn(2, 9, 80, generator=gen) * 2 - 6
    z = torch.randn(2, 8, 9 * STEPS, generator=gen)
    with torch.no_grad():
        want = O.batched(clone(g).double().to(DEV), mels.double().to(DEV), ol, z.double().to(DEV)).float().cpu()
    v = vocoder(g, "3xf16")
    audio, _ = v(mels.to(DEV), torch.tensor(ol, device=DEV), z=z.to(DEV))
    check_gate("3xf16", audio.cpu(), want, torch.tensor(ol), "C=512")


@pytest.mark.parametrize("mode", ["3xf16", "f16"])
def test_audio_matches_oracle_at_the_smallest_channel_count(mode):
    """C = 64, the smallest n_channels the vocoder accepts: 2C = 128 rows of the in-layer output are narrower than the
    640 cond channels, so the plane modes keep the upsampled mels in a workspace region of their own."""
    g = make_oracle(64, 5)
    gen = torch.Generator().manual_seed(6)
    ol = [23, 1, 9]
    mels = torch.randn(3, 23, 80, generator=gen) * 2 - 6
    z = torch.randn(3, 8, 23 * STEPS, generator=gen)
    with torch.no_grad():
        want = O.batched(clone(g).double().to(DEV), mels.double().to(DEV), ol, z.double().to(DEV)).float().cpu()
    v = vocoder(g, mode)
    audio, _ = v(mels.to(DEV), torch.tensor(ol, device=DEV), z=z.to(DEV))
    check_gate(mode, audio.cpu(), want, torch.tensor(ol), "C=64")


def test_sigma_scales_z_with_one_rounding(case, vocoders):
    """The flows receive fp32(sigma * z), the product taken in double: sigma = 0.6 (not an fp32 value) on z gives the
    bits of sigma = 1 on fp32(0.6 * z)."""
    _, _, mels, olens, z, _ = case
    v = vocoders["3xf16"]
    m, ol = mels.to(DEV), olens.to(DEV)
    a, _ = v(m, ol, sigma=0.6, z=z.to(DEV))
    b, _ = v(m, ol, sigma=1.0, z=(z.double() * 0.6).float().to(DEV))
    assert torch.equal(bits(a), bits(b))


@pytest.mark.parametrize("mode", ["3xf16", "fp32"])
def test_round_trip_through_the_oracle_forward(case, vocoders, mode):
    g, g64, mels, _, _, _ = case
    T = 24
    t = torch.arange(T * HOP, dtype=torch.float64) / 22050
    audio = 0.3 * torch.sin(2 * np.pi * 220 * t) + 0.1 * torch.sin(2 * np.pi * 660 * t + 1.0)
    mel = mels[0, :T].double()
    with torch.no_grad():
        z = g64.forward(mel.T[None].to(DEV), audio[None].to(DEV))
    got, _ = vocoders[mode](mels[:1, :T].to(DEV).contiguous(), torch.tensor([T], device=DEV), z=z.float())
    err = float((got[0].double().cpu() - audio).abs().max())
    print(f"\nwaveglow round trip {mode}: max-abs {err:.3e} (|z| max {float(z.abs().max()):.2f})")
    assert err <= 1e-3, err


def test_sigma_zero_is_the_oracle_without_noise(case, vocoders):
    _, g64, mels, olens, z, _ = case
    with torch.no_grad():
        want = O.batched(g64, mels.double().to(DEV), OLENS, torch.zeros_like(z).double().to(DEV), sigma=0.0).float().cpu()
    got, _ = vocoders["3xf16"](mels.to(DEV), olens.to(DEV), sigma=0.0, seed=5)
    check_gate("3xf16", got.cpu(), want, olens, "sigma=0")


@pytest.mark.parametrize("mode", MODES)
def test_per_utterance_bit_identity(case, vocoders, mode):
    _, _, mels, olens, z, _ = case
    v = vocoders[mode]
    m, ol, zz = mels.to(DEV), olens.to(DEV), z.to(DEV)
    B = len(OLENS)
    seeds = torch.arange(100, 100 + B, device=DEV)
    a_z, alens = v(m, ol, z=zz)
    a_s, _ = v(m, ol, seed=seeds)
    rev_z, _ = v(m.flip(0).contiguous(), ol.flip(0).contiguous(), z=zz.flip(0).contiguous())
    rev_s, _ = v(m.flip(0).contiguous(), ol.flip(0).contiguous(), seed=seeds.flip(0).contiguous())
    nan_m, nan_z = m.clone(), zz.clone()
    for b, n in enumerate(OLENS):
        nan_m[b, n:] = float("nan")                                # frames past olens[b] are never read
        nan_z[b, :, n * STEPS:] = float("nan")                     # nor z steps past olens[b] * 32
    assert torch.equal(bits(v(nan_m, ol, z=nan_z)[0]), bits(a_z)), mode
    assert torch.equal(bits(v(nan_m, ol, seed=seeds)[0]), bits(a_s)), mode
    for b, n in enumerate(OLENS):
        one_z, l1 = v(m[b: b + 1, :n].contiguous(), ol[b: b + 1], z=zz[b: b + 1, :, : n * STEPS].contiguous())
        one_s, _ = v(m[b: b + 1, :n].contiguous(), ol[b: b + 1], seed=seeds[b: b + 1])
        assert int(l1[0]) == n * HOP == int(alens[b])
        for batch, rev, one in ((a_z, rev_z, one_z), (a_s, rev_s, one_s)):
            assert torch.equal(bits(batch[b, : n * HOP]), bits(one[0])), (mode, b)
            assert torch.equal(bits(rev[B - 1 - b, : n * HOP]), bits(one[0])), (mode, b)
            assert torch.all(batch[b, n * HOP:] == 0) and not bool(torch.signbit(batch[b, n * HOP:]).any()), (mode, b)
    assert torch.isfinite(a_z).all() and torch.isfinite(a_s).all()


def test_seeded_noise_is_the_noise_tensor(case, vocoders):
    _, _, mels, olens, _, _ = case
    v = vocoders["3xf16"]
    m, ol = mels.to(DEV), olens.to(DEV)
    for seed in (7, torch.tensor([3, -1, 2 ** 62, 0, 5], device=DEV)):
        z = WaveGlowVocoder.noise(ol, m.shape[1], seed)
        assert z.shape == (len(OLENS), 8, m.shape[1] * STEPS)
        for b, n in enumerate(OLENS):
            assert torch.all(z[b, :, n * STEPS:] == 0)
        a, _ = v(m, ol, seed=seed, sigma=0.7)
        b_, _ = v(m, ol, z=z, sigma=0.7)
        assert torch.equal(bits(a), bits(b_))
    # an int seed s gives utterance b the seed s + b
    assert torch.equal(WaveGlowVocoder.noise(ol, m.shape[1], 7), WaveGlowVocoder.noise(ol, m.shape[1], torch.arange(7, 12, device=DEV)))
    # None: one int64 from torch's CPU generator
    torch.manual_seed(11)
    a1, _ = v(m, ol)
    a2, _ = v(m, ol)
    torch.manual_seed(11)
    a3, _ = v(m, ol)
    assert not torch.equal(a1, a2) and torch.equal(bits(a1), bits(a3))


def test_noise_depends_only_on_seed_channel_and_step():
    ol = torch.tensor([40, 3, 17], device=DEV)
    seeds = torch.tensor([5, 6, 7], device=DEV)
    z = WaveGlowVocoder.noise(ol, 40, seeds)
    for b in range(3):
        n = int(ol[b]) * STEPS
        alone = WaveGlowVocoder.noise(ol[b: b + 1], int(ol[b]), seeds[b: b + 1])
        longer = WaveGlowVocoder.noise(ol[b: b + 1], 90, seeds[b: b + 1])
        assert torch.equal(bits(z[b, :, :n]), bits(alone[0])) and torch.equal(bits(longer[0, :, :n]), bits(alone[0]))
    assert not torch.equal(z[0, :, :96], z[1, :, :96])


def test_noise_is_standard_normal():
    from scipy import stats
    z = WaveGlowVocoder.noise(torch.tensor([4000], device=DEV), 4000, 123).flatten().double().cpu().numpy()
    ks = stats.kstest(z, "norm")
    print(f"\nwaveglow noise: {z.size} draws, mean {z.mean():.2e} std {z.std():.4f} KS {ks.statistic:.2e} p {ks.pvalue:.3f}")
    assert ks.pvalue > 1e-3 and abs(z.mean()) < 5e-3 and abs(z.std() - 1) < 5e-3
    for ch in range(8):                                          # every channel, not only the pool
        assert stats.kstest(z.reshape(8, -1)[ch], "norm").pvalue > 1e-4, ch


def test_range_overflow_is_reported_not_clipped(case):
    g, _, mels, olens, z, _ = case
    sd = dict(g.state_dict())
    sd["WN.11.start.weight_g"] = sd["WN.11.start.weight_g"] * 1e5          # the first WN's x far beyond 4094
    for mode in ("f16", "3xf16"):
        v = WaveGlowVocoder(256, math_mode=mode)
        v.load_state_dict(sd)
        with pytest.raises(ValueError, match="range"):
            v.to(DEV)(mels.to(DEV), olens.to(DEV), z=z.to(DEV))
    v = WaveGlowVocoder(256, math_mode="fp32")
    v.load_state_dict(sd)
    v.to(DEV)(mels.to(DEV), olens.to(DEV), z=z.to(DEV))


def test_bad_lengths_raise(case, vocoders):
    _, _, mels, _, z, _ = case
    for bad in ([0, 1, 2, 3, 4], [65, 1, 2, 3, 4]):
        with pytest.raises(ValueError, match="olens"):
            vocoders["3xf16"](mels.to(DEV), torch.tensor(bad, device=DEV), z=z.to(DEV))


# prep, noise, upsampling operand and GEMM, (cond planes,) then per flow: start, 8 x (cond GEMM, in-layer GEMM, gate,
# skip GEMM), 7 res GEMMs, the flow kernel
@pytest.mark.parametrize("mode,launches", [("3xf16", 4 + 1 + 12 * 41), ("f16", 4 + 1 + 12 * 41), ("tf32", 4 + 12 * 41),
                                           ("fp32", 496)])
def test_graph_capture_replays_bit_identically_and_launch_count(case, vocoders, mode, launches):
    _, _, mels, olens, _, _ = case
    v = vocoders[mode]
    m, ol = mels.to(DEV), olens.to(DEV)
    B, L = m.shape[:2]
    seeds = torch.arange(B, device=DEV)
    audio = torch.empty(B, L * HOP, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    h = v._handle(m.device)
    ws = v._workspace(h, B, L, m.device)
    lib = _lib.load()

    def call():
        _lib.check(lib.fs2_waveglow(h, _lib.ptr(m), _lib.ptr(ol), B, L, 1.0, _lib.ptr(seeds), None, _lib.ptr(audio), _lib.ptr(status),
                                    _lib.ptr(ws), ws.numel(), _lib.stream_ptr(m.device)), "fs2_waveglow")

    before = lib.fs2_kernel_launches()
    call()
    assert lib.fs2_kernel_launches() - before == launches
    torch.cuda.synchronize()
    eager = audio.clone()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):                 # the call allocates nothing and never synchronises
        call()
    audio.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    assert torch.equal(bits(audio), bits(eager))


def test_dropin_hub_checkpoint_matches_oracle(case, tmp_path, monkeypatch):
    g, g64, mels, _, z, _ = case
    plain = O.WaveGlow.remove_weightnorm(clone(g))
    sd = {"module." + k: v for k, v in plain.state_dict().items()}
    assert any(k.endswith("start.weight") for k in sd) and not any(k.endswith("weight_g") for k in sd)
    path = tmp_path / "waveglow.pt"
    torch.save({"state_dict": sd, "epoch": 0}, path)
    monkeypatch.setattr(torch.hub, "load", lambda *a, **k: pytest.fail("the network hub must not be reached"))
    dropin_run.install_waveglow_hub(str(path))
    waveglow = torch.hub.load("nvidia/DeepLearningExamples:torchhub", "nvidia_waveglow", model_math="fp32")
    waveglow = waveglow.remove_weightnorm(waveglow)
    waveglow = waveglow.to(DEV).eval()
    assert waveglow.math_mode == "3xf16" and waveglow.n_channels == 256
    n = 37
    got, _ = waveglow(mels[:1, :n].to(DEV).contiguous(), torch.tensor([n], device=DEV), z=z[:1, :, : n * STEPS].to(DEV).contiguous())
    with torch.no_grad():
        want = g64.infer(mels[0, :n].double().T[None].to(DEV), 1.0, z[:1, :, : n * STEPS].double().to(DEV)).float().cpu()
    check_gate("3xf16", got.cpu(), want, torch.tensor([n]), "hub checkpoint")
    audio = waveglow.infer(mels[:1, :n].transpose(1, 2).contiguous().to(DEV), sigma=0.6)     # the notebook's call
    assert audio.shape == (1, n * HOP) and torch.isfinite(audio).all()


def test_end_to_end_from_synthesize():
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
    audio, alens = v(mels, olens, sigma=0.6, seed=1)
    B, L = mels.shape[:2]
    assert audio.shape == (B, L * HOP) and audio.dtype == torch.float32
    assert torch.equal(alens, olens * HOP)
    assert torch.isfinite(audio).all()
    for b in range(B):
        assert torch.all(audio[b, int(alens[b]):] == 0)
        one, _ = v(mels[b: b + 1, : int(olens[b])].contiguous(), olens[b: b + 1], sigma=0.6, seed=1 + b)
        assert torch.equal(bits(one[0]), bits(audio[b, : int(alens[b])])), b
