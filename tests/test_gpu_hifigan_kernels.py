"""HiFi-GAN's own layers (csrc/hifigan.cu) against float64, one at a time, through fs2_op_hifigan_resblock and
fs2_op_hifigan_upsample, which run fs2_hifigan's packing and launch code for that layer:

  * both residual block types at every (C, k, dilations) that V1 (ResBlock1) and V3 (ResBlock2) use, in all four modes;
  * every upsampling (Cin, Cout, u) of V1 and V3, in all four modes;
  * ragged lens including 0 and 1, rows per utterance not a multiple of 16; rows past lens +0 with no sign bit, NaN in the
    input rows past lens inert; sentinel guard bands around every output; the range bit of the status word.

Gates are relative to the size of the summed terms: the error of an output element over sum |term| of the float64 layer
(through every convolution of a block), against the float64 operands ("exact") and, in f16 / tf32, against the operands
those modes multiply (fp16 hi planes at scale 16 and the weights at their power-of-two scale; tf32-truncated fp32).
Gate values are at most 3x the errors measured on an H100 (DESIGN.md section 16)."""
import zlib

import pytest
import torch
import torch.nn.functional as F

from fastspeech2_b200 import _lib
from test_gpu_tap_gemm import MODE, TF32_CONVERSION, Guarded, bits, f16_operands, to_tf32

DEV = "cuda"
MODES = ("fp32", "tf32", "f16", "3xf16")
RANGE = _lib.FS2_HIFIGAN_RANGE
LP = 45                                   # rows per utterance: not a multiple of 16
LENS = (0, 1, LP, 37, LP - 3)
# (type, C, k, dilations): V1's ResBlock1 at every stage width and kernel size, V3's ResBlock2 likewise
BLOCKS = ([(1, C, k, (1, 3, 5)) for C in (256, 128, 64, 32) for k in (3, 7, 11)] +
          [(2, C, k, d) for C in (128, 64, 32) for k, d in ((3, (1, 2)), (5, (2, 6)), (7, (3, 12)))])
UPSAMPLES = [(512, 256, 8), (256, 128, 8), (128, 64, 2), (64, 32, 2),         # V1
             (128, 64, 8), (64, 32, 4)]                                        # V3 (its first stage is V1's second)
# (max, mean) of the relative error per layer kind, mode and label: 3x the largest value measured over the cases on an
# H100 80GB HBM3, rounded down.  ResBlock1's six chained convolutions make its sum of |terms| large, so its ratios are small.
GATES = {
    "rb1": {"fp32": {"exact": (1.4e-8, 3.2e-11)}, "3xf16": {"exact": (1.4e-8, 3.9e-11)},
            "f16": {"fp16 operands": (1.4e-7, 4e-10), "exact": (1.3e-5, 3.9e-8)},
            "tf32": {"tf32 operands": (1.3e-8, 5.9e-10), "exact": (4.6e-5, 1.4e-7)}},
    "rb2": {"fp32": {"exact": (9.2e-8, 8.7e-9)}, "3xf16": {"exact": (1.9e-7, 2.6e-8)},
            "f16": {"fp16 operands": (4.7e-6, 7.6e-8), "exact": (1.3e-4, 1.4e-5)},
            "tf32": {"tf32 operands": (6.3e-6, 9.6e-8), "exact": (5e-4, 4.4e-5)}},
    "upsample": {"fp32": {"exact": (1.2e-6, 7.5e-8)}, "3xf16": {"exact": (3.8e-6, 5.2e-7)},
                 "f16": {"fp16 operands": (1.6e-6, 1.8e-7), "exact": (6.6e-4, 1.2e-4)},
                 "tf32": {"tf32 operands": (2.8e-6, 3.5e-7), "exact": (1.8e-3, 3.1e-4)}}}


def lrelu(v):
    return F.leaky_relu(v, 0.1)


def q16(v):
    """The hi plane of an activation, back in fp32: rn_fp16(16 v) / 16."""
    return (v.float() * 16).clamp(-65504, 65504).half().float() / 16


def q16w(w):
    """A weight at its power-of-two scale, rounded to fp16 (what the hi weight plane holds)."""
    return f16_operands(w[:1].flatten(), w)[1]


def tf32(v):
    return to_tf32(v.float().contiguous(), TF32_CONVERSION)


def operands(label):
    """(activation rounding, weight rounding) of a reference"""
    return {"exact": (lambda v: v, lambda w: w), "fp16 operands": (q16, q16w), "tf32 operands": (tf32, tf32)}[label]


def valid(lens, L):
    return torch.arange(L, device=DEV)[None, :] < torch.as_tensor(lens, device=DEV)[:, None]


def rel_error(got, want, terms, mask):
    e = ((got.double() - want).abs() / terms.clamp_min(1e-30))[mask]
    return (float(e.max()), float(e.mean())) if e.numel() else (0.0, 0.0)


def block_reference(x, lens, type_, k, dils, ws, bs, act, qa, qw):
    """float64 residual block per utterance on [B, Lp, C] (zero padding at each utterance's edges, zeros past lens): act
    the leaky ReLU (identity for the terms), qa / qw the rounding of every conv's input / weight."""
    out = torch.zeros(x.shape, dtype=torch.float64, device=DEV)
    conv = lambda w, b, v, d: F.conv1d(qa(v).double(), qw(w).double(), b.double(), dilation=d, padding=d * (k - 1) // 2)
    for i, n in enumerate(lens):
        if n == 0:
            continue
        y = x[i, :n].double().T[None]
        for m, d in enumerate(dils):
            if type_ == 1:
                y = conv(ws[3 + m], bs[3 + m], act(conv(ws[m], bs[m], act(y), d)), 1) + y
            else:
                y = conv(ws[m], bs[m], act(y), d) + y
        out[i, :n] = y[0].T
    return out


def upsample_reference(x, lens, w, b, u, act, qa, qw):
    B, Lin, _ = x.shape
    out = torch.zeros(B, Lin * u, w.shape[1], dtype=torch.float64, device=DEV)
    for i, n in enumerate(lens):
        if n:
            out[i, : n * u] = F.conv_transpose1d(qa(act(x[i, :n].double())).double().T[None], qw(w).double(), b.double(), stride=u,
                                                 padding=u // 2)[0].T
    return out


def run_block(mode, type_, C, k, dils, x, lens, ws, bs):
    import ctypes as Ct
    lib = _lib.load()
    B, Lp, _ = x.shape
    g = Guarded(B * Lp * C, torch.float32)
    status = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    d = (Ct.c_int * len(dils))(*dils)
    wp = (Ct.c_void_p * len(ws))(*[t.data_ptr() for t in ws])
    bp = (Ct.c_void_p * len(bs))(*[t.data_ptr() for t in bs])
    _lib.check(lib.fs2_op_hifigan_resblock(MODE[mode], type_, C, k, len(dils), d, _lib.ptr(x), _lib.ptr(lens), B, Lp, wp, bp,
                                           _lib.ptr(g.view), _lib.ptr(status), _lib.stream_ptr(x.device)), "fs2_op_hifigan_resblock")
    torch.cuda.synchronize()
    assert g.intact(), f"{mode}: a store landed outside the output"
    return g.view.view(B, Lp, C), int(status.item())


def run_upsample(mode, Cin, Cout, u, x, lens, w, b):
    lib = _lib.load()
    B, Lin, _ = x.shape
    g = Guarded(B * Lin * u * Cout, torch.float32)
    status = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    _lib.check(lib.fs2_op_hifigan_upsample(MODE[mode], Cin, Cout, u, _lib.ptr(x), _lib.ptr(lens), B, Lin, _lib.ptr(w), _lib.ptr(b),
                                           _lib.ptr(g.view), _lib.ptr(status), _lib.stream_ptr(x.device)), "fs2_op_hifigan_upsample")
    torch.cuda.synchronize()
    assert g.intact(), f"{mode}: a store landed outside the output"
    return g.view.view(B, Lin * u, Cout), int(status.item())


def block_data(type_, C, k, dils):
    """Seeded x [B, LP, C] ~ N(0, 0.5^2) on every row; weights in torch layouts at the scale of a weight-normed conv."""
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(f"{type_}-{C}-{k}-{dils}".encode()))
    x = torch.randn(len(LENS), LP, C, generator=gen, device=DEV) * 0.5
    n = 6 if type_ == 1 else 2
    ws = [torch.randn(C, C, k, generator=gen, device=DEV) / (k * C) ** 0.5 for _ in range(n)]
    bs = [torch.randn(C, generator=gen, device=DEV) * 0.1 for _ in range(n)]
    return x, torch.tensor(LENS, dtype=torch.int64, device=DEV), ws, bs


def _check(mode, gates, out, ref, terms, mask, what):
    failed = []
    for label, (gmax, gmean) in gates[mode].items():
        mx, mn = rel_error(out, ref(*operands(label)), terms, mask)
        print(f"GATE {mode:5s} {what:26s} {label:14s} max {mx:.3e} / {gmax:.0e}  mean {mn:.3e} / {gmean:.0e}")
        if not (mx <= gmax and mn <= gmean):
            failed.append((label, mx, mn))
    assert not failed, (mode, what, failed)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("type_,C,k,dils", BLOCKS, ids=[f"rb{t}-C{C}-k{k}-d{'.'.join(map(str, d))}" for t, C, k, d in BLOCKS])
def test_resblock_vs_float64(mode, type_, C, k, dils):
    x, lens, ws, bs = block_data(type_, C, k, dils)
    mask = valid(LENS, LP)
    out, status = run_block(mode, type_, C, k, dils, x, lens, ws, bs)
    assert status == 0
    assert bool((bits(out)[~mask] == 0).all()), "rows past lens are not +0"
    xn = x.masked_fill(~mask[..., None], float("nan"))
    out_n, status_n = run_block(mode, type_, C, k, dils, xn, lens, ws, bs)
    assert status_n == 0 and torch.equal(bits(out_n), bits(out)), "NaN past lens reached the output"
    terms = block_reference(x.abs(), LENS, type_, k, dils, [w.abs() for w in ws], [b.abs() for b in bs], lambda v: v.abs(),
                            lambda v: v, lambda w: w)
    ref = lambda qa, qw: block_reference(x, LENS, type_, k, dils, ws, bs, lrelu, qa, qw)
    _check(mode, GATES[f"rb{type_}"], out, ref, terms, mask, f"rb{type_} C{C} k{k} d{dils}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("Cin,Cout,u", UPSAMPLES, ids=[f"{a}-{b}-u{u}" for a, b, u in UPSAMPLES])
def test_upsample_vs_float64(mode, Cin, Cout, u):
    gen = torch.Generator(device=DEV).manual_seed(Cin * 31 + u)
    x = torch.randn(len(LENS), LP, Cin, generator=gen, device=DEV) * 0.5
    w = torch.randn(Cin, Cout, 2 * u, generator=gen, device=DEV) / (2 * Cin) ** 0.5
    b = torch.randn(Cout, generator=gen, device=DEV) * 0.1
    lens = torch.tensor(LENS, dtype=torch.int64, device=DEV)
    out, status = run_upsample(mode, Cin, Cout, u, x, lens, w, b)
    assert status == 0
    mask = valid([n * u for n in LENS], LP * u)
    assert bool((bits(out)[~mask] == 0).all()), "rows past lens * u are not +0"
    xn = x.masked_fill(~valid(LENS, LP)[..., None], float("nan"))
    assert torch.equal(bits(run_upsample(mode, Cin, Cout, u, xn, lens, w, b)[0]), bits(out)), "NaN past lens reached the output"
    terms = upsample_reference(x, LENS, w.abs(), b.abs(), u, lambda v: lrelu(v).abs(), lambda v: v, lambda w: w)
    ref = lambda qa, qw: upsample_reference(x, LENS, w, b, u, lrelu, qa, qw)
    _check(mode, GATES["upsample"], out, ref, terms, mask, f"upsample {Cin}->{Cout} u{u}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_range_bit(mode):
    """An input past +-4094 in one utterance sets FS2_HIFIGAN_RANGE in f16 / 3xf16, never in fp32 / tf32."""
    x, lens, ws, bs = block_data(2, 64, 3, (1, 2))
    x[3] *= 2e4
    want = RANGE if mode in ("f16", "3xf16") else 0
    assert run_block(mode, 2, 64, 3, (1, 2), x, lens, ws, bs)[1] == want
    assert run_upsample(mode, 64, 32, 4, x, lens, torch.randn(64, 32, 8, device=DEV) * 0.1, torch.zeros(32, device=DEV))[1] == want
