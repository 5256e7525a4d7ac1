"""MelGAN's own kernels (csrc/melgan.cu) against float64, one layer at a time, through fs2_op_melgan_block and
fs2_op_melgan_upsample, which run fs2_melgan's code for that layer:

  * every residual block instantiation: C in {32, 64, 128, 256} x dilation {1, 3, 9}, the unfused route (producers +
    tap-GEMMs) in all four modes and the fused melgan_block_kernel in f16 and 3xf16, all 8 of its instantiations
    (C = 256 stages h through shared memory; C = 128 and 256 loop over column groups);
  * the polyphase transposed convolution of each of the four upsampling stages, in all four modes;
  * ragged batches: an empty utterance, one of d + 1 rows (reflection at both edges of every row), one of Lp rows, Lp
    not a multiple of 16 (one warp's 16 rows span two live utterances) and B * Lp not a multiple of a CTA's rows (the
    last CTA has a partial warp and warps that return at once);
  * rows past lens: +0 with no sign bit, and NaN in the input rows past lens changes no output bit;
  * sentinel guard bands around every output, and the range bit of the status word.

Gates are relative to the size of the summed terms: the error of an output element over sum |term| of the float64
block (through both of its layers), and each mode has its own reference operands.  The tight gates compare against the
operands the kernels multiply (fp16 hi planes at scale 16 and the weights at their power-of-two scale in f16, tf32-
truncated fp32 in tf32), the exact gates against the float64 operands.  Gate values are small multiples of the errors
measured on an H100 (DESIGN.md section 8).  The two routes are held to agree within the tight gate; on an H100 they
came out bit-identical in every case."""
import zlib
from dataclasses import dataclass
from typing import Tuple

import pytest
import torch
import torch.nn.functional as F

from fastspeech2_b200 import _lib
from test_gpu_tap_gemm import MODE, TF32_CONVERSION, Guarded, bits, f16_operands, to_tf32

DEV = "cuda"
MODES = ("fp32", "tf32", "f16", "3xf16")
CHANNELS = (32, 64, 128, 256)
DILATIONS = (1, 3, 9)
UNFUSED, FUSED = 1, 2
ROUTES = {"fp32": (UNFUSED,), "tf32": (UNFUSED,), "f16": (UNFUSED, FUSED), "3xf16": (UNFUSED, FUSED)}
ROUTE_NAME = {UNFUSED: "unfused", FUSED: "fused"}
RANGE = _lib.FS2_MELGAN_RANGE


# ---- restatement of the launch geometry (melgan.cu) ------------------------------------------------------------------
def warps(C):
    """melgan_block_kernel's warps per CTA; each warp owns 16 rows."""
    return 2 if C == 256 else 4


def fused_blocks(mode, C):
    """The route fs2_melgan takes: fused in f16 at C <= 128 and in 3xf16 at C <= 64."""
    return (mode == "f16" and C <= 128) or (mode == "3xf16" and C <= 64)


@dataclass(frozen=True)
class BlockCase:
    C: int
    d: int
    Lp: int
    lens: Tuple[int, ...]

    @property
    def B(self):
        return len(self.lens)

    @property
    def name(self):
        return f"C{self.C}-d{self.d}-Lp{self.Lp}"

    @property
    def rows(self):
        return self.B * self.Lp


def straddles(c):
    """Warps whose 16 rows hold live rows of two utterances."""
    out = []
    for m0 in range(0, c.rows, 16):
        live = {m // c.Lp for m in range(m0, min(m0 + 16, c.rows)) if m % c.Lp < c.lens[m // c.Lp]}
        if len(live) > 1:
            out.append(m0)
    return out


def last_cta(c):
    """(rows of the last CTA, warps of it with no row at all)."""
    per = 16 * warps(c.C)
    rem = c.rows % per or per
    return rem, warps(c.C) - -(-rem // 16)


def _block_case(C, d, i):
    """Lp = 29 + 16 k + 2 i (never a multiple of 16); lengths Lp, d + 1, 0, then values in [d + 1, Lp]; B >= 5, the first
    with a last CTA that has a partial warp and a warp without rows."""
    Lp = 29 + 16 * DILATIONS.index(d) + 2 * i
    B = 5
    while True:
        rem, idle = last_cta(BlockCase(C, d, Lp, (0,) * B))
        if rem % 16 and idle:
            break
        B += 1
    lens = [Lp, d + 1, 0] + [d + 1 + (7 * k + i) % (Lp - d) for k in range(B - 3)]
    return BlockCase(C, d, Lp, tuple(lens))


BLOCK_CASES = [_block_case(C, d, i) for i, C in enumerate(CHANNELS) for d in DILATIONS]
# (Cin, Cout, s) of the four ConvTranspose1d stages
UPSAMPLE_STAGES = ((512, 256, 8), (256, 128, 8), (128, 64, 2), (64, 32, 2))
UPSAMPLE_LIN, UPSAMPLE_LENS = 150, (150, 0, 1, 77, 129)     # 150 = a 128-row tile + a tail; 77 and 129 tails of their own


def check_coverage():
    """What the block cases must reach; returns the list of what they miss."""
    miss = []
    for mode in MODES:
        for route in ROUTES[mode]:
            for C in CHANNELS:
                if not any(c.C == C for c in BLOCK_CASES):
                    miss.append(f"{mode} {ROUTE_NAME[route]} C={C}")
    fused = {(C, mode) for mode in ("f16", "3xf16") if FUSED in ROUTES[mode] for C in CHANNELS if any(c.C == C for c in BLOCK_CASES)}
    if len(fused) != 8:
        miss.append(f"fused instantiations reached: {sorted(fused)}")
    for C in CHANNELS:
        if {c.d for c in BLOCK_CASES if c.C == C} != set(DILATIONS):
            miss.append(f"C={C}: dilations")
    for c in BLOCK_CASES:
        if not all(n == 0 or c.d + 1 <= n <= c.Lp for n in c.lens):
            miss.append(f"{c.name}: a length outside {{0}} u [d + 1, Lp]")
        for n, what in ((0, "empty"), (c.d + 1, "d + 1"), (c.Lp, "Lp")):
            if n not in c.lens:
                miss.append(f"{c.name}: no {what} utterance")
        if c.Lp % 16 == 0 or not straddles(c):
            miss.append(f"{c.name}: no warp spans two live utterances")
        rem, idle = last_cta(c)
        if rem % 16 == 0 or idle == 0:
            miss.append(f"{c.name}: the last CTA has no partial warp or no idle warp")
    for n in (0, 1):
        if n not in UPSAMPLE_LENS:
            miss.append(f"upsampling: no length {n}")
    if not any(n % 128 and n > 128 for n in UPSAMPLE_LENS):
        miss.append("upsampling: no tile tail after a full tile")
    return miss


# ---- references --------------------------------------------------------------------------------------------------
def lrelu(v):
    return F.leaky_relu(v, 0.2)


def q16(v):
    """The hi plane of an activation, back in fp32: rn_fp16(16 v) / 16."""
    return (v.float() * 16).clamp(-65504, 65504).half().float() / 16


def q16w(w):
    """A weight at its power-of-two scale, rounded to fp16 (what the hi weight plane holds)."""
    return f16_operands(w[:1].flatten(), w)[1]


def tf32(v):
    return to_tf32(v.float(), TF32_CONVERSION)


def block_reference(xs, xa, lens, d, w1, b1, w2, b2, ws, bs, act, q2):
    """float64 residual block per utterance, [B, Lp, C]; xs the shortcut operand, xa the dilated conv's (after lrelu), act
    on h, q2 the rounding of lrelu(h); zeros past lens."""
    out = torch.zeros(xs.shape, dtype=torch.float64, device=DEV)
    w1, b1, w2, b2, ws, bs = (t.double() for t in (w1, b1, w2, b2, ws, bs))
    for b, n in enumerate(lens):
        if n == 0:
            continue
        a = xa[b, :n].double().T[None]
        h = F.conv1d(F.pad(a, (d, d), mode="reflect"), w1, b1, dilation=d)
        y = F.conv1d(q2(act(h)).double(), w2, b2) + F.conv1d(xs[b, :n].double().T[None], ws, bs)
        out[b, :n] = y[0].T
    return out


def block_gates(mode, x, w):
    """(label, reference block arguments, max gate, mean gate) per gate; w = (w1, b1, w2, b2, ws, bs)."""
    w1, b1, w2, b2, ws, bs = w
    exact = (x, lrelu(x), w1, b1, w2, b2, ws, bs, lrelu, lambda v: v)
    C = x.shape[-1]
    if mode == "fp32":
        return [("exact", exact, 2e-7, 2e-8)]
    if mode == "3xf16":
        return [("exact", exact, 5e-7, 5e-8)]
    if mode == "f16":
        pair = q16w(torch.cat([w2, ws], 1))                       # [W2 | Ws] shares one scale
        ops = (q16(x), q16(lrelu(x)), q16w(w1), b1, pair[:, :C].contiguous(), b2, pair[:, C:].contiguous(), bs, lrelu, q16)
        return [("fp16 operands", ops, 3e-5, 2e-7), ("exact", exact, 3e-4, 5e-5)]
    ops = (tf32(x), tf32(lrelu(x)), tf32(w1), b1, tf32(w2), b2, tf32(ws), bs, lrelu, tf32)
    return [("tf32 operands", ops, 4e-5, 4e-7), ("exact", exact, 8e-4, 2e-4)]


def block_terms(x, lens, d, w):
    """sum |term| of each output element through both layers: |Ws| |x| + |W2| (|W1| * |lrelu(x)| + |b1|) + |b2| + |bs|."""
    w1, b1, w2, b2, ws, bs = (t.abs() for t in w)
    return block_reference(x.abs(), lrelu(x).abs(), lens, d, w1, b1, w2, b2, ws, bs, lambda v: v, lambda v: v)


def valid(lens, L):
    return torch.arange(L, device=DEV)[None, :] < torch.as_tensor(lens, device=DEV)[:, None]


def rel_error(got, want, terms, mask):
    e = ((got.double() - want).abs() / terms.clamp_min(1e-30))[mask]
    return (float(e.max()), float(e.mean())) if e.numel() else (0.0, 0.0)


# ---- calls -------------------------------------------------------------------------------------------------------
def run_block(mode, route, c, x, lens, w):
    """One fs2_op_melgan_block call on a sentinel-guarded output; -> (out [B, Lp, C], status).  The call's kernel count
    tells the routes apart: the fused one launches 3 kernels fewer than the unfused one (1 against taps, GEMM, concat,
    GEMM)."""
    lib = _lib.load()
    w1, b1, w2, b2, ws, bs = w
    g = Guarded(c.rows * c.C, torch.float32)
    status = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    run_block.launches = lib.fs2_kernel_launches()
    rc = lib.fs2_op_melgan_block(MODE[mode], route, c.C, _lib.ptr(x), _lib.ptr(lens), c.B, c.Lp, c.d, _lib.ptr(w1), _lib.ptr(b1),
                                 _lib.ptr(w2), _lib.ptr(b2), _lib.ptr(ws), _lib.ptr(bs), _lib.ptr(g.view), _lib.ptr(status),
                                 _lib.stream_ptr(x.device))
    _lib.check(rc, "fs2_op_melgan_block")
    run_block.launches = lib.fs2_kernel_launches() - run_block.launches
    torch.cuda.synchronize()
    assert g.intact(), f"{mode} {ROUTE_NAME.get(route, route)}: a store landed outside the output"
    return g.view.view(c.B, c.Lp, c.C), int(status.item())


def run_upsample(mode, Cin, Cout, s, x, lens, w, b):
    lib = _lib.load()
    B, Lin, _ = x.shape
    g = Guarded(B * Lin * s * Cout, torch.float32)
    status = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    rc = lib.fs2_op_melgan_upsample(MODE[mode], Cin, Cout, s, _lib.ptr(x), _lib.ptr(lens), B, Lin, _lib.ptr(w), _lib.ptr(b),
                                    _lib.ptr(g.view), _lib.ptr(status), _lib.stream_ptr(x.device))
    _lib.check(rc, "fs2_op_melgan_upsample")
    torch.cuda.synchronize()
    assert g.intact(), f"{mode}: a store landed outside the output"
    return g.view.view(B, Lin * s, Cout), int(status.item())


def block_data(c):
    """Seeded x [B, Lp, C] ~ N(0, 0.5^2) on every row, weights in torch layouts at the scale of a weight-normed conv."""
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(c.name.encode()))
    C = c.C
    x = torch.randn(c.B, c.Lp, C, generator=gen, device=DEV) * 0.5
    w = (torch.randn(C, C, 3, generator=gen, device=DEV) / (3 * C) ** 0.5, torch.randn(C, generator=gen, device=DEV) * 0.1,
         torch.randn(C, C, 1, generator=gen, device=DEV) / C ** 0.5, torch.randn(C, generator=gen, device=DEV) * 0.1,
         torch.randn(C, C, 1, generator=gen, device=DEV) / C ** 0.5, torch.randn(C, generator=gen, device=DEV) * 0.1)
    return x, torch.tensor(c.lens, dtype=torch.int64, device=DEV), w


# ---- GPU tests -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("c", BLOCK_CASES, ids=[c.name for c in BLOCK_CASES])
def test_block_vs_float64(mode, c):
    """Each route of the mode against float64 per gate, +0 past lens, NaN past lens inert, status 0; in f16 / 3xf16 the
    two routes agree within the tight gate and route 0 is the route fs2_melgan takes."""
    x, lens, w = block_data(c)
    mask = valid(c.lens, c.Lp)
    terms = block_terms(x, c.lens, c.d, w)
    gates = [(label, block_reference(*args[:2], c.lens, c.d, *args[2:]), gmax, gmean) for label, args, gmax, gmean in block_gates(mode, x, w)]
    xn = x.masked_fill(~mask[..., None], float("nan"))
    got, failed, launches = {}, [], {}
    for route in ROUTES[mode]:
        out, status = run_block(mode, route, c, x, lens, w)
        launches[route] = run_block.launches
        rname = ROUTE_NAME[route]
        assert status == 0, (mode, rname, status)
        assert bool((bits(out)[~mask] == 0).all()), f"{mode} {rname}: rows past lens are not +0"
        for label, want, gmax, gmean in gates:
            mx, mn = rel_error(out, want, terms, mask)
            print(f"GATE {mode:5s} {c.name:18s} {rname:7s} {label:14s} max {mx:.3e} / {gmax:.0e}  mean {mn:.3e} / {gmean:.0e}")
            if not (mx <= gmax and mn <= gmean):
                failed.append((rname, label, mx, mn))
        out_n, status_n = run_block(mode, route, c, xn, lens, w)
        assert status_n == 0 and torch.equal(bits(out_n), bits(out)), f"{mode} {rname}: NaN past lens reached the output"
        got[route] = out
    assert not failed, (mode, c.name, failed)
    if len(got) == 2:
        assert launches[UNFUSED] - launches[FUSED] == 3, launches
        mx, _ = rel_error(got[FUSED], got[UNFUSED].double(), terms, mask)
        print(f"GATE {mode:5s} {c.name:18s} fused vs unfused    max {mx:.3e} / {gates[0][2]:.0e}")
        assert mx <= gates[0][2], (mode, c.name, mx)
        out0, _ = run_block(mode, 0, c, x, lens, w)
        assert torch.equal(bits(out0), bits(got[FUSED if fused_blocks(mode, c.C) else UNFUSED])), "route 0 is not fs2_melgan's route"


UPSAMPLE_GATES = {"fp32": [("exact", 1.5e-6, 1e-7)], "3xf16": [("exact", 5e-6, 5e-7)],
                  "f16": [("fp16 operands", 2e-6, 2e-7), ("exact", 8e-4, 1.5e-4)],
                  "tf32": [("tf32 operands", 3e-6, 4e-7), ("exact", 1.5e-3, 4e-4)]}


def upsample_reference(xa, lens, w, b, s, Lout):
    """float64 ConvTranspose1d(k = 2s, stride s, padding s/2) of xa (after lrelu) per utterance; zeros past lens * s."""
    B, _, _ = xa.shape
    out = torch.zeros(B, Lout, w.shape[1], dtype=torch.float64, device=DEV)
    for i, n in enumerate(lens):
        if n:
            out[i, : n * s] = F.conv_transpose1d(xa[i, :n].double().T[None], w.double(), b.double(), stride=s, padding=s // 2)[0].T
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("Cin,Cout,s", UPSAMPLE_STAGES, ids=[f"{a}-{b}-s{s}" for a, b, s in UPSAMPLE_STAGES])
def test_upsample_vs_float64(mode, Cin, Cout, s):
    """The polyphase GEMM (pack kind 1) against float64 conv_transpose1d per utterance, +0 past lens * s, NaN inert."""
    gen = torch.Generator(device=DEV).manual_seed(Cin * 31 + s)
    B, Lin, lens = len(UPSAMPLE_LENS), UPSAMPLE_LIN, UPSAMPLE_LENS
    x = torch.randn(B, Lin, Cin, generator=gen, device=DEV) * 0.5
    w = torch.randn(Cin, Cout, 2 * s, generator=gen, device=DEV) / (2 * Cin) ** 0.5
    b = torch.randn(Cout, generator=gen, device=DEV) * 0.1
    lt = torch.tensor(lens, dtype=torch.int64, device=DEV)
    out, status = run_upsample(mode, Cin, Cout, s, x, lt, w, b)
    assert status == 0
    mask = valid([n * s for n in lens], Lin * s)
    assert bool((bits(out)[~mask] == 0).all()), "rows past lens * s are not +0"
    terms = upsample_reference(lrelu(x).abs(), lens, w.abs(), b.abs(), s, Lin * s)
    ops = {"exact": (lrelu(x), w), "fp16 operands": (q16(lrelu(x)), q16w(w)), "tf32 operands": (tf32(lrelu(x)), tf32(w))}
    failed = []
    for label, gmax, gmean in UPSAMPLE_GATES[mode]:
        mx, mn = rel_error(out, upsample_reference(*ops[label][:1], lens, ops[label][1], b, s, Lin * s), terms, mask)
        print(f"GATE {mode:5s} upsample {Cin:3d}->{Cout:3d} s{s} {label:14s} max {mx:.3e} / {gmax:.0e}  mean {mn:.3e} / {gmean:.0e}")
        if not (mx <= gmax and mn <= gmean):
            failed.append((label, mx, mn))
    assert not failed, (mode, Cin, failed)
    xn = x.masked_fill(~valid(lens, Lin)[..., None], float("nan"))
    assert torch.equal(bits(run_upsample(mode, Cin, Cout, s, xn, lt, w, b)[0]), bits(out)), "NaN past lens reached the output"


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_range_bit(mode):
    """x past +-4094 in one utterance sets FS2_MELGAN_RANGE on every route of f16 / 3xf16, and never in fp32 / tf32."""
    c = next(c for c in BLOCK_CASES if c.C == 64 and c.d == 3)
    x, lens, w = block_data(c)
    x[3] *= 2e4
    want = RANGE if mode in ("f16", "3xf16") else 0
    for route in ROUTES[mode]:
        _, status = run_block(mode, route, c, x, lens, w)
        assert status == want, (mode, ROUTE_NAME[route], status)
    Cin, Cout, s = UPSAMPLE_STAGES[3]
    xu = torch.randn(2, 20, Cin, device=DEV)
    xu[1] *= 2e4
    _, status = run_upsample(mode, Cin, Cout, s, xu, torch.tensor([20, 11], device=DEV), torch.randn(Cin, Cout, 2 * s, device=DEV) * 0.1,
                             torch.zeros(Cout, device=DEV))
    assert status == want, (mode, "upsample", status)
