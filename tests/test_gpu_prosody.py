"""Prosody controls (speed, pitch, energy) on the H100, in every precision mode: neutral factors change nothing, a
controlled batch stays bit-identical per utterance to the B = 1 call with its slice of the controls, the duration
arithmetic and the fp32 multiply on pitch / energy are exact at the C ABI, and B = 1 matches the CPU oracle.
Needs an H100: run with `-m gpu`."""
import math

import pytest
import torch

import _prosody_oracle as P
from fastspeech2_b200 import _lib
from fastspeech2_b200 import length_regulator as LR
from fastspeech2_b200.serving import export_torchscript
from test_gpu_parity import PRECISIONS, TOL, close
from test_gpu_per_utterance import ILENS, build, ragged

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def models(weights):
    return {prec: build(weights, prec) for prec in PRECISIONS}


def controls(il, T, seed=5):
    """Distinct factors: speed per phoneme, pitch per utterance (semitones), energy per phoneme."""
    g = torch.Generator().manual_seed(seed)
    B = len(il)
    speed = 0.6 + torch.rand(B, T, generator=g)                                    # 0.6 .. 1.6
    pitch = 2.0 ** (torch.randint(-6, 7, (B,), generator=g).float() / 12)
    energy = 0.5 + torch.rand(B, T, generator=g)
    return speed, pitch, energy


@pytest.mark.parametrize("prec", PRECISIONS)
def test_neutral_controls_bit_identical(models, prec):
    """Explicit all-1.0 factors take the control path through every kernel and change no bit."""
    m = models[prec]
    xs, il = ragged(ILENS)
    ones = torch.ones(xs.shape, device="cuda")
    with torch.no_grad():
        want = m.synthesize(xs.cuda(), il.cuda())
        got = m.synthesize(xs.cuda(), il.cuda(), speed=ones, pitch=ones, energy=ones)
        got_b = m.synthesize(xs.cuda(), il.cuda(), speed=1.0, pitch=torch.ones(len(ILENS)), energy=None)
    for w, g, gb in zip(want, got, got_b):
        assert torch.equal(w, g) and torch.equal(w, gb)
    for b in (0, 2, 5):
        n = ILENS[b]
        x = xs[b, :n].cuda()
        with torch.no_grad():
            plain = m.inference(x)
            ctl = m.inference_controlled(x, speed=torch.ones(n, device="cuda"), pitch=1.0, energy=torch.ones(n))
        assert torch.equal(plain, ctl), b


def check_independent(m, xs, il, speed, pitch, energy):
    with torch.no_grad():
        mels, olens, dur = m.synthesize(xs.cuda(), il.cuda(), speed=speed.cuda(), pitch=pitch.cuda(), energy=energy.cuda())
    assert torch.equal(dur.sum(1), olens) and mels.shape[1] == int(olens.max())
    for b, n in enumerate(il.tolist()):
        L = int(olens[b])
        with torch.no_grad():
            want = m.inference_controlled(xs[b, :n].cuda(), speed=speed[b, :n].cuda(), pitch=pitch[b].cuda(),
                                          energy=energy[b, :n].cuda())
        assert want.shape[0] == L, (b, want.shape, L)
        assert torch.equal(mels[b, :L], want), f"mels of utterance {b}: max diff {(mels[b, :L] - want).abs().max():.3e}"
        assert not mels[b, L:].any() and not dur[b, n:].any(), f"padding of utterance {b}"
    return mels, olens, dur


@pytest.mark.parametrize("prec", PRECISIONS)
def test_controlled_batch_independent_of_batch_mates(models, prec):
    m = models[prec]
    xs, il = ragged(ILENS)
    speed, pitch, energy = controls(ILENS, xs.shape[1])
    mels, olens, dur = check_independent(m, xs, il, speed, pitch, energy)
    with torch.no_grad():
        plain = m.synthesize(xs.cuda(), il.cuda())
    assert not torch.equal(dur, plain[2])                   # the speeds moved some durations
    r = torch.arange(len(ILENS) - 1, -1, -1)
    mels_r, olens_r, dur_r = check_independent(m, xs[r], il[r], speed[r], pitch[r], energy[r])
    for b in range(len(ILENS)):
        L = int(olens[b])
        assert int(olens_r[r[b]]) == L and torch.equal(dur_r[r[b]], dur[b]) and torch.equal(mels_r[r[b], :L], mels[b, :L])


def unit_duration_model(weights, prec):
    """Duration head that predicts exactly 1 everywhere: round(exp(log 2) - 1) = 1."""
    sd = {k: v.clone() for k, v in weights.items()}
    sd["duration_predictor.linear.weight"].zero_()
    sd["duration_predictor.linear.bias"].fill_(math.log(2.0))
    return build(sd, prec)


def host_rule(speed, il):
    """rint_half_even(fp32(1) * fp32(a)), then all-zero -> all-one per utterance, 0 past ilens."""
    d = torch.round(torch.ones_like(speed) * speed.float()).long()
    d[torch.arange(speed.shape[1])[None, :] >= il[:, None]] = 0
    d[d.sum(1) == 0] = (torch.arange(speed.shape[1])[None, :] < il[d.sum(1) == 0][:, None]).long()
    return d


@pytest.mark.parametrize("prec", PRECISIONS)
def test_exact_duration_arithmetic(weights, prec):
    m = unit_duration_model(weights, prec)
    xs, il = ragged(ILENS, seed=3)
    valid = (torch.arange(xs.shape[1])[None, :] < il[:, None]).long()
    with torch.no_grad():
        _, olens, dur = m.synthesize(xs.cuda(), il.cuda())
        assert torch.equal(dur.cpu(), valid)
        for s, k in ((2.5, 2), (3.5, 4), (0.4, 1)):          # half-even ties; 0.4 rounds all to 0 -> the all-ones rule
            _, olens, dur = m.synthesize(xs.cuda(), il.cuda(), speed=s)
            assert torch.equal(dur.cpu(), k * valid) and torch.equal(olens.cpu(), k * il), s
        g = torch.Generator().manual_seed(9)
        table = torch.tensor([0.4, 0.5, 0.7, 1.1, 1.5, 2.5, 3.5, 4.49])
        speed = table[torch.randint(0, len(table), xs.shape, generator=g)]
        speed[1, :] = 0.4                                    # utterance 1 (one phoneme) falls back to all ones
        _, olens, dur = m.synthesize(xs.cuda(), il.cuda(), speed=speed.cuda())
    want = host_rule(speed, il)
    assert torch.equal(dur.cpu(), want) and torch.equal(olens.cpu(), want.sum(1))


def test_frame_count_overflow_raises(weights):
    """A scaled utterance past the int32 prefix sum of the length plan raises instead of wrapping."""
    sd = {k: v.clone() for k, v in weights.items()}
    sd["duration_predictor.linear.weight"].zero_()
    sd["duration_predictor.linear.bias"].fill_(math.log(1e6 + 1))     # ~1e6 frames per phoneme
    m = build(sd, "3xf16")
    xs, il = ragged([3, 5])
    with torch.no_grad(), pytest.raises(ValueError, match="int32 prefix sum"):
        m.synthesize(xs.cuda(), il.cuda(), speed=torch.tensor([1.0, 1e4]))
    hs = torch.zeros(2, 5, 4, device="cuda")
    ds = torch.full((2, 5), 1 << 20, dtype=torch.int64, device="cuda")
    alpha = torch.tensor([[1.0] * 5, [1e30] * 5], device="cuda")
    _, olens, stats, _ = LR.plan(hs, ds, torch.tensor([5, 5]), alpha_v=alpha)
    assert olens[0].item() == 5 << 20 and olens[1].item() >= 2 ** 31 and stats[0].item() == olens[1].item()


def decode(m, hm, olens, flags, e_scale=None, p_scale=None, es=None):
    """fs2_decode_ctl on a given hm -> (return code, after, e_out, p_out, e_ids, p_ids)."""
    lib = _lib.load()
    h = m._ready(hm)
    B, L, _ = hm.shape
    ws = m._ws(B, 1, L)
    f32 = dict(dtype=torch.float32, device="cuda")
    before, after = torch.empty(B, L, 80, **f32), torch.empty(B, L, 80, **f32)
    e_out, p_out = torch.empty(B, L, **f32), torch.empty(B, L, **f32)
    e_ids, p_ids = (torch.empty(B, L, dtype=torch.int64, device="cuda") for _ in range(2))
    P_ = _lib.ptr
    rc = lib.fs2_decode_ctl(h, P_(hm), P_(olens), P_(es), P_(es), B, L, P_(before), P_(after), P_(e_out), P_(p_out),
                            P_(e_ids), P_(p_ids), P_(e_scale), P_(p_scale), P_(ws), ws.numel(), flags,
                            _lib.stream_ptr(hm.device))
    return rc, after, e_out, p_out, e_ids, p_ids


@pytest.mark.parametrize("prec", PRECISIONS)
def test_exact_pitch_energy_at_the_abi(models, prec):
    m = models[prec]
    g = torch.Generator().manual_seed(4)
    il = torch.tensor([11, 7, 16])
    B, T = len(il), int(il.max())
    hs = (torch.randn(B, T, 256, generator=g) * 0.5).cuda()
    ds = torch.randint(0, 5, (B, T), generator=g)
    ds[:, 0] = 2
    ds[1, 3:] = 0                                                   # zero-duration phonemes, one all-but-first
    ds[torch.arange(T)[None, :] >= il[:, None]] = 0
    fac_in = 0.5 + torch.rand(2, B, T, generator=g)
    cum, olens, stats, il_dev = LR.plan(hs, ds.cuda(), il)
    L = int(stats[0]) + 3                                           # frames past every olens
    fac_out = torch.empty(2, B, L, device="cuda")
    hm = LR.gather(hs, cum, il_dev, L, fac_in.cuda().contiguous(), fac_out)
    assert torch.equal(hm, LR.gather(hs, cum, il_dev, L))
    for b in range(B):
        n, ol = int(il[b]), int(olens[b])
        for k in range(2):
            want = torch.repeat_interleave(fac_in[k, b, :n], ds[b, :n])
            assert torch.equal(fac_out[k, b, :ol].cpu(), want) and bool((fac_out[k, b, ol:] == 1.0).all()), (k, b)
    e_bins, p_bins = m.energy_predictor.energy_bins, m.pitch_predictor.pitch_bins
    for flags in (0, _lib.FS2_PER_UTTERANCE):
        ol_arg = olens if flags else None
        rc0, after0, e0, p0, _, _ = decode(m, hm, ol_arg, flags)
        rc1, after1, e1, p1, ei1, pi1 = decode(m, hm, ol_arg, flags, fac_out[0], fac_out[1])
        assert rc0 == 0 and rc1 == 0
        assert torch.equal(e1, e0 * fac_out[0]) and torch.equal(p1, p0 * fac_out[1]), flags
        valid = (torch.arange(L, device="cuda")[None, :] < olens[:, None]) if flags else torch.ones_like(e1, dtype=torch.bool)
        assert torch.equal(ei1[valid], torch.bucketize(e1, e_bins)[valid]) and torch.equal(pi1[valid], torch.bucketize(p1, p_bins)[valid])
        assert not torch.equal(after0, after1)                          # the factors reach the decoder
    rc, *_ = decode(m, hm, olens, _lib.FS2_PER_UTTERANCE, fac_out[0], None, es=torch.zeros(B, L, device="cuda"))
    assert rc == -1                                                 # FS2_ERR_INVALID: scales need predict mode


@pytest.mark.parametrize("prec", PRECISIONS)
def test_controlled_inference_against_oracle(models, weights, prec):
    """B = 1 against the CPU oracle: durations and bucket ids exact, mels within TOL."""
    m = models[prec]
    x = torch.randint(1, 68, (23,), generator=torch.Generator().manual_seed(13))
    n = x.shape[0]
    g = torch.Generator().manual_seed(8)
    cases = [(1.1, 2 ** (3 / 12), 1.1), (2.5, 2 ** (-5 / 12), 0.8),
             (0.7 + torch.rand(n, generator=g), 0.8 + 0.4 * torch.rand(n, generator=g), 0.6 + torch.rand(n, generator=g))]
    for s, p, e in cases:
        with torch.no_grad():
            got = m.inference_controlled(x.cuda(), speed=s, pitch=p, energy=e)
            _, want, used, e_ids, p_ids, _, _ = P.inference_path(weights, x[None], torch.tensor([n]), P.per_phoneme(s, n),
                                                                 P.per_phoneme(p, n), P.per_phoneme(e, n))
            _, after_b, dur_b, oh_e, oh_p = m._forward(x[None].cuda(), torch.tensor([n]).cuda(), is_inference=True,
                                                       _controls=(P.per_phoneme(s, n).cuda(), P.per_phoneme(p, n).cuda(),
                                                                  P.per_phoneme(e, n).cuda()))
        want = want[0]
        assert torch.equal(after_b[0], got)
        assert torch.equal(dur_b[0].cpu(), used[0])
        assert torch.equal(oh_e[0].argmax(-1).cpu(), e_ids[0]) and torch.equal(oh_p[0].argmax(-1).cpu(), p_ids[0])
        close(got, want, TOL[prec], f"controlled mel ({prec})")


def test_served_synthesize_controlled_matches_model(tmp_path, models):
    m = models["3xtf32"]
    served = torch.jit.load(export_torchscript(m, str(tmp_path / "fs2.pt"))).cuda()
    xs, il = ragged(ILENS)
    speed, pitch, energy = (t.cuda() for t in controls(ILENS, xs.shape[1], seed=6))
    with torch.no_grad():
        want = m.synthesize(xs.cuda(), il.cuda(), speed=speed, pitch=pitch, energy=energy)
    got = served.synthesize_controlled(xs.cuda(), il.cuda(), speed, pitch, energy)
    for w, g in zip(want, got):
        assert torch.equal(w, g)
    one = torch.ones((), device="cuda")
    neutral = served.synthesize_controlled(xs.cuda(), il.cuda(), one, one, one)
    plain = served.synthesize(xs.cuda(), il.cuda())
    assert torch.equal(neutral[0], plain[0]) and torch.equal(neutral[1], plain[1])
