"""The tap GEMM (gemm_tc.cu's tap_gemm_tc_kernel and gemm_fp32.cu) against float64, through fs2_op_tap_gemm_ex.

The tensor-core kernel is persistent: grid = min(tiles, SMs), CTA c walks tiles c, c + grid, ..., and its k-th tile
belongs to consumer warpgroup k & 1.  Whether the second warpgroup, the order barriers, a ring that carries over from one
tile to the next, dead tiles or packed tails run at all depends on the shape, so this file restates the kernel's schedule
in Python (tile width, ring depth, tiling, tile coordinates, the walk) and chooses its cases with it.  The CPU tests
assert what the case table covers on a 132-SM H100; the GPU tests assert the same for the device they run on, then
check the numbers:

  * every case against a float64 conv1d / matmul (then act, then residual), with per-family gates;
  * per-utterance mode (lens): bit-identity with B = 1 calls and with the batch reversed, exact zeros past lens in out
    and in every plane, NaN padding that changes nothing, transposed-V entries past lens or L never written;
  * schedule independence: an utterance alone (one tile per CTA, warpgroup 0 only) and inside a batch of more than
    2 x SMs tiles (some of its tiles on warpgroup 1) gives the same bits;
  * the epilogue's operand planes bit for bit against a restatement of split_pair, and the transposed V third bit for
    bit against the plain output;
  * guard bands of sentinel bits around every output.
"""
import math
import zlib
from dataclasses import dataclass
from typing import Optional, Tuple

import pytest
import torch
import torch.nn.functional as F

from fastspeech2_b200 import _lib

# ---- restatement of the kernel's schedule (gemm_tc.cu) ------------------------------------------------------------
H100_SMS = 132
BM = 128
RING_BUDGET = 227 * 1024 - 1024 - 256       # shared memory for the ring: 227 KB less alignment slack and barriers
TC_FAMILIES = ("tf32", "f16", "3xf16")      # tap_gemm_tc_kernel<BN, PRECISE, HALF>: <., false, false>, <., false, true>, <., true, true>
FAMILIES = ("fp32",) + TC_FAMILIES          # fp32: the CUDA-core kernel of gemm_fp32.cu
WIDTHS = (128, 80, 64, 32, 16)
MODE = {"fp32": _lib.MATH_FP32, "tf32": _lib.MATH_TF32, "f16": _lib.MATH_F16, "3xf16": _lib.MATH_3XTF32}
PLANES = {"f16": 1, "3xf16": 2}             # operand planes the plane families write (hi; hi + lo)


def tile_width(N):
    """Widest tile that divides N (wgmma N = 128, 64 + 16, 64, 16 + 16, 16)."""
    return 128 if N % 128 == 0 else 80 if N % 80 == 0 else 64 if N % 64 == 0 else 32 if N % 32 == 0 else 16


def bke(fam):
    """K elements per pipeline step: one 128-byte swizzle row of fp32 (tf32) or fp16 (the plane families)."""
    return 32 if fam == "tf32" else 64


def stages(fam, bn):
    """Cfg<BN, PRECISE, HALF>::STAGES: A (128 x 128 B) + B (BN x 128 B) per stage, hi + lo in 3xF16, at most 8."""
    stage = (2 if fam == "3xf16" else 1) * (BM * 128 + bn * 128)
    return min(8, RING_BUDGET // stage)


def steps_per_tile(fam, K, taps):
    return taps * -(-K // bke(fam))


@dataclass(frozen=True)
class Tiling:
    flat: bool
    B: int
    full: int        # ordinary 128-row tiles per utterance
    gn: int          # 16-row granules of an utterance's tail
    upt: int         # utterances per packed tail tile
    m_tiles: int
    n_tiles: int

    @property
    def full_tiles(self):
        return self.full * self.B

    @property
    def total(self):
        return self.m_tiles * self.n_tiles

    @property
    def packed(self):
        return self.m_tiles > self.full_tiles


def tiling(B, L, N, taps, per_utt):
    """launch(): flat [B*L, K] for plain GEMMs without lens, else per utterance: floor(L / 128) full tiles and the tails
    (L % 128 rows, gn granules of 16) of upt utterances packed into shared tiles; a tail over 64 rows is one more
    ordinary tile."""
    n_tiles = N // tile_width(N)
    if taps == 1 and not per_utt:
        return Tiling(True, 1, 0, 1, 1, -(-(B * L) // BM), n_tiles)
    full, tail = L // BM, L % BM
    gn = -(-tail // 16) if tail else 1
    upt = 8 // gn if tail else 1
    if tail and upt == 1:
        full, tail, gn = full + 1, 0, 1
    return Tiling(False, B, full, gn, upt, full * B + (-(-B // upt) if tail else 0), n_tiles)


def tile_coords(t, tile, lens):
    """(utterance, first row, packed index or -1, dead) of a tile, as the kernel's tile_coords."""
    mt = tile // t.n_tiles
    if t.flat:
        b, t0, packed = 0, mt * BM, -1
    elif mt < t.full_tiles:
        b, t0, packed = mt // t.full, (mt % t.full) * BM, -1
    else:
        packed = mt - t.full_tiles
        b, t0 = packed * t.upt, t.full * BM
    return b, t0, packed, packed < 0 and lens is not None and t0 >= lens[b]


def walk(t, lens, sms):
    """The persistent walk: CTA c takes tiles c, c + grid, ...; its k-th tile goes to warpgroup k & 1.
    Returns one list per CTA of (tile, dead)."""
    grid = min(t.total, sms)
    return [[(tile, tile_coords(t, tile, lens)[3]) for tile in range(c, t.total, grid)] for c in range(grid)]


# ---- cases -------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Case:
    name: str
    B: int
    L: int
    K: int
    N: int
    taps: int
    act: int = 0                         # 0 none, 1 ReLU, 2 tanh
    bias: bool = True
    resid: bool = False
    wscale: float = 1.0                  # weights, bias and residual times this power of two (act is none / ReLU)
    lens: Optional[Tuple[int, ...]] = None

    def tiling(self):
        return tiling(self.B, self.L, self.N, self.taps, self.lens is not None)


N_BY_WIDTH = {16: (16, 48), 32: (32, 96), 64: (64, 192), 80: (80, 160, 240), 128: (128, 384)}


def _schedule_cases(fam):
    """Five cases per tile width: steps per tile 1, S - 1, S, S + 1 and >= 4 S (S = ring depth), each with one of the
    three tile counts that matter to the walk: at most one tile per CTA, SMs + 1 (one CTA gets a second tile, on
    warpgroup 1), more than 2 x SMs with an odd count on some CTAs."""
    E = bke(fam)
    out = []
    for i, bn in enumerate(WIDTHS):
        S = stages(fam, bn)
        Ns = N_BY_WIDTH[bn]

        def k_for(steps, taps, partial):
            return (steps // taps) * E - (16 if partial else 0)

        def odd_divisor(s, options):
            return next(tp for tp in options if s % tp == 0)

        t1 = odd_divisor(S - 1, (3, 1))
        t2 = odd_divisor(S, (7, 5, 3, 1))
        t3 = odd_divisor(S + 1, (9, 5, 3, 1))
        many = -(-4 * S // 9)
        w3 = N_BY_WIDTH[bn][-1]
        # tiles: > 2 SMs, flat: ceil(4 * 2840 / 128) = 89 row tiles x 3 column tiles = 267
        out.append(Case(f"{fam}-bn{bn}-steps1", 4, 2840, E - 16 * (i % 2), w3, 1, act=i % 3, bias=True, resid=i % 2 == 0))
        # SMs + 1: 19 utterances x 7 full tiles, or ceil(7 * 2420 / 128) = 133 flat row tiles
        shape = (19, 896) if t1 > 1 else (7, 2420)
        out.append(Case(f"{fam}-bn{bn}-steps{S - 1}", *shape, k_for(S - 1, t1, i % 2 == 1), bn, t1, act=(i + 1) % 3,
                        bias=i % 2 == 1, resid=True))
        # one tile per CTA: 13 utterances of 40 rows (L < 128: a packed conv whose boxes start at row -pad)
        out.append(Case(f"{fam}-bn{bn}-steps{S}", 13, 40, k_for(S, t2, i % 2 == 0), Ns[0], t2, act=(i + 2) % 3,
                        bias=i % 2 == 0, resid=i % 2 == 1))
        # > 2 SMs: 89 row tiles x 3 column tiles, or 133 x 2 (N = 160)
        n3 = Ns[1]
        shape = (89, 128) if n3 // bn == 3 else (133, 128)
        if t3 == 1:
            shape = (1, shape[0] * 128 - 5)
        out.append(Case(f"{fam}-bn{bn}-steps{S + 1}", *shape, k_for(S + 1, t3, i % 2 == 1), n3, t3,
                        act=1 if bn == 64 else i % 3,
                        bias=i % 2 == 1, resid=i % 2 == 0, wscale=2.0 ** 10 if bn == 64 else 1.0))
        # many ring rounds per tile, one tile per CTA: 3 utterances of 300 rows (2 full tiles and packed tails of 44 rows)
        out.append(Case(f"{fam}-bn{bn}-steps{9 * many}", 3, 300, k_for(9 * many, 9, i % 2 == 0), Ns[-1], 9,
                        act=1 if bn == 32 else (i + 1) % 3, bias=True, resid=i % 2 == 1,
                        wscale=2.0 ** -10 if bn == 32 else 1.0))
    return out


FP32_CASES = [
    Case("fp32-conv9", 3, 70, 256, 1024, 9, act=1, resid=True),
    Case("fp32-flat", 2, 333, 384, 384, 1, bias=False),
    Case("fp32-conv5-tanh", 5, 41, 80, 240, 5, act=2, resid=True),
    Case("fp32-conv3", 4, 100, 208, 48, 3, bias=False, resid=True, act=1),
    Case("fp32-w2^10", 2, 130, 560, 96, 1, act=1, resid=True, wscale=2.0 ** 10),
    Case("fp32-w2^-10", 3, 50, 64, 160, 3, act=0, resid=False, wscale=2.0 ** -10),
]
SCHEDULE_CASES = {"fp32": FP32_CASES, **{fam: _schedule_cases(fam) for fam in TC_FAMILIES}}

# Per-utterance mode; every case runs in every family.  The two walk cases put dead tiles where the walk needs them
# (per_utterance_coverage): 36 utterances x 8 ordinary tiles = 288 tiles, and 20 x 5 x 3 column tiles = 300 tiles.
PER_UTT_CASES = [
    Case("walk-flat", 36, 1000, 208, 128, 1, act=1, resid=True,
         lens=(991, 864, 988, 414, 597, 47, 15, 142, 0, 310, 929, 1000, 17, 516, 523, 776, 802, 488, 223, 849, 394, 1,
               366, 41, 911, 257, 497, 129, 940, 127, 913, 255, 430, 33, 49, 265)),
    Case("walk-conv9", 20, 600, 80, 240, 9, act=2,
         lens=(127, 257, 414, 497, 15, 600, 47, 430, 49, 41, 255, 0, 394, 129, 310, 17, 523, 33, 1, 265)),
    Case("tail-gn1", 13, 140, 560, 48, 5, resid=True, lens=(140, 0, 127, 129, 17, 15, 140, 1, 33, 31, 128, 12, 100)),
    Case("tail-gn2", 6, 160, 80, 96, 3, act=1, bias=False, lens=(160, 128, 0, 49, 47, 130)),
    Case("tail-gn3-short", 5, 40, 208, 64, 9, act=2, resid=True, lens=(40, 0, 17, 39, 1)),
    Case("tail-gn4", 3, 180, 80, 160, 1, resid=True, lens=(180, 63, 65)),
    Case("tail-over64", 4, 200, 208, 192, 5, act=1, resid=True, lens=(200, 129, 0, 127)),
]
# the q|k|v projections of the encoder (C = 256, d_k = 128) and decoder (C = 384, d_k = 192), 2 heads; L = 1 (mod 8) so
# that the transposed rows have a padded tail [L, lpad)
VT_CASES = [
    Case("qkv-enc", 3, 257, 256, 768, 1, lens=(257, 0, 100)),
    Case("qkv-dec", 2, 385, 384, 1152, 1, lens=(130, 385)),
    Case("qkv-dec-full", 2, 201, 384, 1152, 1),
]
VT_HEADS = 2
# one utterance alone, and the same utterances as a batch of 12 x 8 x 3 = 288 tiles
INDEPENDENCE_CASES = [Case("batch-conv3", 12, 1000, 208, 384, 3, act=1, resid=True),
                      Case("batch-flat", 12, 1000, 208, 384, 1, act=2)]


def lpad_of(L):
    return (L + 7) // 8 * 8


# ---- what the table covers -----------------------------------------------------------------------------------------
def schedule_coverage(sms):
    """Per tensor-core instantiation (family, tile width): the tile counts and steps per tile its cases reach."""
    got = {}
    for fam in TC_FAMILIES:
        for c in SCHEDULE_CASES[fam]:
            t, bn = c.tiling(), tile_width(c.N)
            S, s = stages(fam, bn), steps_per_tile(fam, c.K, c.taps)
            counts = [len(w) for w in walk(t, None, sms)]
            facts = got.setdefault((fam, bn), set())
            if t.total <= sms:
                facts.add("one tile per CTA")
            if t.total == sms + 1:
                facts.add("SMs + 1 tiles")
            if t.total > 2 * sms and any(n % 2 for n in counts):
                facts.add("> 2 x SMs tiles, odd count on a CTA")
            facts.add("1 step" if s == 1 else "< ring depth" if s < S else "= ring depth" if s == S else
                      "ring depth + 1" if s == S + 1 else ">= 4 x ring depth" if s >= 4 * S else "other")
    return got


SCHEDULE_FACTS = {"one tile per CTA", "SMs + 1 tiles", "> 2 x SMs tiles, odd count on a CTA", "1 step", "< ring depth",
                  "= ring depth", "ring depth + 1", ">= 4 x ring depth"}


def per_utterance_coverage(sms):
    facts = set()
    for c in PER_UTT_CASES:
        t = c.tiling()
        for cta in walk(t, c.lens, sms):
            dead = [d for _, d in cta]
            for k in range(len(dead) - 1):
                if dead[k] and not dead[k + 1]:
                    facts.add(f"dead tile at {'odd' if k % 2 else 'even'} k, then a live tile")
                if dead[k] and dead[k + 1]:
                    facts.add("two consecutive dead tiles")
            if dead and dead[-1]:
                facts.add("a CTA's last tile is dead")
        if 0 in c.lens:
            facts.add("lens 0")
        if c.L in c.lens:
            facts.add("lens L")
        if any(n > 16 and n % 16 in (1, 15) for n in c.lens):
            facts.add("lens 16 g +- 1")
        if 127 in c.lens and 129 in c.lens:
            facts.add("lens 127 and 129")
    return facts


PER_UTTERANCE_FACTS = {"dead tile at odd k, then a live tile", "dead tile at even k, then a live tile",
                       "two consecutive dead tiles", "a CTA's last tile is dead", "lens 0", "lens L", "lens 16 g +- 1",
                       "lens 127 and 129"}


def tiling_coverage(cases):
    facts = set()
    for c in cases:
        t = c.tiling()
        if t.packed:
            facts.add(f"gn {t.gn} upt {t.upt}")
            if c.B % t.upt:
                facts.add("B not a multiple of upt")
        if not t.flat and c.L % BM > 64:
            facts.add("tail over 64 rows")
        facts.add(f"taps {c.taps}")
        if c.taps > 1 and c.L < BM:
            facts.add("conv with L < 128")
    return facts


TILING_FACTS = {"gn 1 upt 8", "gn 2 upt 4", "gn 3 upt 2", "gn 4 upt 2", "tail over 64 rows", "B not a multiple of upt",
                "taps 1", "taps 3", "taps 5", "taps 9", "conv with L < 128"}


def epilogue_coverage(fam):
    cases = SCHEDULE_CASES[fam] + PER_UTT_CASES
    facts = {f"act {c.act}" for c in cases} | {f"bias {c.bias}" for c in cases} | {f"resid {c.resid}" for c in cases}
    facts |= {f"wscale {c.wscale}" for c in cases}
    facts |= {f"N {c.N}" for c in cases}
    if fam != "fp32":
        facts |= {"K whole steps" if c.K % bke(fam) == 0 else "K % BKE != 0" for c in cases}
    return facts


def epilogue_facts(fam):
    want = {"act 0", "act 1", "act 2", "bias True", "bias False", "resid True", "resid False", f"wscale {2.0 ** 10}",
            f"wscale {2.0 ** -10}"}
    if fam != "fp32":
        want |= {"K whole steps", "K % BKE != 0"} | {f"N {n}" for ns in N_BY_WIDTH.values() for n in ns}
    return want


def independence_coverage(sms):
    facts = set()
    for c in INDEPENDENCE_CASES:
        alone = tiling(1, c.L, c.N, c.taps, False)
        if alone.total <= sms:
            facts.add("alone: one tile per CTA")
        t = c.tiling()
        if t.total > 2 * sms:
            for cta in walk(t, None, sms):
                if any(k % 2 for k, _ in enumerate(cta)):
                    facts.add("batch: tiles on warpgroup 1")
    return facts


def check_coverage(sms):
    missing = []
    for key, facts in sorted(schedule_coverage(sms).items()):
        missing += [(key, f) for f in SCHEDULE_FACTS - facts]
    if {k for k in schedule_coverage(sms)} != {(f, bn) for f in TC_FAMILIES for bn in WIDTHS}:
        missing.append("not every (family, tile width) instantiation")
    missing += [("per utterance", f) for f in PER_UTTERANCE_FACTS - per_utterance_coverage(sms)]
    for fam in FAMILIES:
        cases = SCHEDULE_CASES[fam] + PER_UTT_CASES
        want = TILING_FACTS if fam != "fp32" else {"taps 1", "taps 3", "taps 5", "taps 9", "conv with L < 128"}
        missing += [(fam, f) for f in want - tiling_coverage(cases)]
        missing += [(fam, f) for f in epilogue_facts(fam) - epilogue_coverage(fam)]
        for c in cases:      # tight gates were set at depths up to 3456
            if c.K * c.taps > 3456:
                missing.append((fam, c.name, "K * taps > 3456"))
    missing += [("independence", f) for f in {"alone: one tile per CTA", "batch: tiles on warpgroup 1"} - independence_coverage(sms)]
    for c in VT_CASES:
        if c.L % 8 != 1:
            missing.append((c.name, "L % 8 != 1"))
    if {(c.N, (c.N // 3) // VT_HEADS) for c in VT_CASES} != {(768, 128), (1152, 192)}:
        missing.append("transposed V at N = 768 / dk 128 and N = 1152 / dk 192")
    return missing


def test_case_table_covers_the_schedule():
    """On a 132-SM H100: every instantiation, tile count, ring depth, dead-tile pattern and packed tail listed above."""
    assert check_coverage(H100_SMS) == []


def test_schedule_restatement():
    """Spot values of the restated schedule: ring depths per family and tile width, tails, dead tiles."""
    assert [stages("tf32", bn) for bn in WIDTHS] == [7, 8, 8, 8, 8]
    assert [stages("f16", bn) for bn in WIDTHS] == [7, 8, 8, 8, 8]
    assert [stages("3xf16", bn) for bn in WIDTHS] == [3, 4, 4, 5, 6]
    tails = [tiling(3, L, 128, 3, False) for L in (140, 160, 180, 190, 200, 40)]
    assert [(t.gn, t.upt, t.full) for t in tails] == [(1, 8, 1), (2, 4, 1), (4, 2, 1), (4, 2, 1), (1, 1, 2), (3, 2, 0)]
    assert tiling(4, 2840, 48, 1, False) == Tiling(True, 1, 0, 1, 1, 89, 3)
    t = tiling(5, 300, 48, 5, True)            # 2 full tiles each, tails of 44 rows: gn 3, two per packed tile
    assert (t.full_tiles, t.m_tiles, t.n_tiles, t.total) == (10, 13, 3, 39)
    assert tile_coords(t, 3 * 11, (300,) * 5) == (2, 256, 1, False)
    assert tile_coords(t, 3 * 3 + 2, (300, 100, 0, 0, 0)) == (1, 128, -1, True)
    assert tile_coords(t, 3 * 2, (300, 100, 0, 0, 0)) == (1, 0, -1, False)
    assert steps_per_tile("tf32", 80, 9) == 27 and steps_per_tile("3xf16", 80, 9) == 18


def test_rejects_bad_arguments_on_the_host():
    """fs2_op_tap_gemm_ex refuses these before it touches memory (the pointers are never dereferenced)."""
    lib = _lib.load()
    p = 256     # a stand-in non-null, aligned pointer

    def call(mode=_lib.MATH_3XTF32, out=p, planes=None, vt=None, vt_col0=512, vt_heads=2, vt_lpad=264, L=257):
        return lib.fs2_op_tap_gemm_ex(mode, p, 2, L, 256, p, None, 768, 1, 0, None, None, out, planes, vt_col0, vt_heads,
                                      vt, vt_lpad, None)
    assert call(mode=_lib.MATH_FP32, planes=p) == -1 and b"out_planes" in lib.fs2_last_error()
    assert call(mode=_lib.MATH_FP32, vt=p) == -1 and b"transposed V" in lib.fs2_last_error()
    assert call(mode=_lib.MATH_TF32, planes=p) == -1 and b"out_planes" in lib.fs2_last_error()
    assert call(mode=_lib.MATH_TF32, out=None, vt=p) == -1 and b"null" in lib.fs2_last_error()
    assert call(mode=7) == -1 and b"math mode" in lib.fs2_last_error()
    assert call(vt=p, vt_heads=0) == -1 and b"vt_col0" in lib.fs2_last_error()
    assert call(vt=p, vt_heads=3, vt_col0=512) == -1 and b"heads" in lib.fs2_last_error()
    assert call(vt=p, vt_col0=768) == -1
    assert call(vt=p, vt_lpad=256) == -1 and b"vt_lpad" in lib.fs2_last_error()
    assert call(L=-1) == -1 and b"shape" in lib.fs2_last_error()
    assert lib.fs2_op_tap_gemm(_lib.MATH_F16, p, 2, 4, 64, p, None, 64, 1, 0, None, None, None) == -1


# ---- GPU: helpers ------------------------------------------------------------------------------------------------
SENT32 = 0x7FA5A5A5          # fp32 NaN payload that no kernel writes
SENT16 = 0x7DA5              # fp16 NaN payload
DEV = "cuda"
PAD = 64                     # guard elements before and after every output (keeps the 32-byte alignment)
# What the H100's tf32 wgmma does to fp32 operands read from shared memory: truncation to the 10-bit mantissa, in A and
# in B, as test_tf32_operand_conversion observed on an H100 80GB HBM3.  The tight tf32 gate compares against operands
# converted this way.
TF32_CONVERSION = "truncate"


class Guarded:
    """An output of n elements in the middle of a buffer filled with sentinel bits; `post` extra elements after it."""

    def __init__(self, n, dtype, post=0):
        self.n, self.post = n, PAD + post
        self.buf = torch.empty(PAD + n + self.post, dtype=dtype, device=DEV)
        self.bits().fill_(SENT32 if dtype == torch.float32 else SENT16)
        self.view = self.buf[PAD:PAD + n]

    def bits(self, t=None):
        t = self.buf if t is None else t
        return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)

    def intact(self):
        s = SENT32 if self.buf.dtype == torch.float32 else SENT16
        return bool((self.bits()[:PAD] == s).all()) and bool((self.bits()[PAD + self.n:] == s).all())


def bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def tap_gemm(fam, x, w, bias, act, resid, lens=None, *, out=True, planes=False, vt=None):
    """One fs2_op_tap_gemm_ex call on sentinel-guarded outputs.  vt = (col0, heads, lpad).  Returns out [B, L, N],
    planes [P, B*L, N] and vt ([B*heads, dk, lpad] fp32, or [P, B*heads, dk, lpad] fp16), each None when not asked for,
    after checking that no byte outside them changed."""
    lib = _lib.load()
    B, L, K = x.shape
    taps, N, _ = w.shape
    P = PLANES.get(fam, 1)
    rows = B * L
    g_out = Guarded(rows * N, torch.float32) if out else None
    # f16 writes the hi plane only: the band after it is as large as a lo plane would be
    g_pl = Guarded(P * rows * N, torch.float16, post=rows * N if P == 1 else 0) if planes else None
    g_vt = None
    if vt is not None:
        col0, heads, lpad = vt
        n_vt = B * (N - col0) * lpad
        g_vt = (Guarded(n_vt, torch.float32) if fam == "tf32" else
                Guarded(P * n_vt, torch.float16, post=n_vt if P == 1 else 0))
    col0, heads, lpad = vt if vt is not None else (0, 0, 0)
    rc = lib.fs2_op_tap_gemm_ex(MODE[fam], _lib.ptr(x), B, L, K, _lib.ptr(w), _lib.ptr(bias), N, taps, act, _lib.ptr(resid),
                                _lib.ptr(lens), _lib.ptr(g_out.view) if out else None,
                                _lib.ptr(g_pl.view) if planes else None, col0, heads,
                                _lib.ptr(g_vt.view) if g_vt is not None else None, lpad, _lib.stream_ptr(x.device))
    _lib.check(rc, "fs2_op_tap_gemm_ex")
    torch.cuda.synchronize()
    for name, g in (("out", g_out), ("planes", g_pl), ("vt", g_vt)):
        assert g is None or g.intact(), f"{fam}: a store landed outside {name}"
    res_vt = None
    if g_vt is not None:
        shape = (B * heads, (N - col0) // heads, lpad)
        res_vt = g_vt.view.view(*shape) if fam == "tf32" else g_vt.view.view(P, *shape)
    return (g_out.view.view(B, L, N) if out else None, g_pl.view.view(P, rows, N) if planes else None, res_vt)


def split_planes(v, P):
    """split_pair restated: hi = rn_fp16(sat(16 v)), lo = rn_fp16(sat(16 v - hi)); int16 bits [P, ...]."""
    a = v.float() * 16
    hi = a.clamp(-65504, 65504).half()
    out = [hi]
    if P == 2:
        out.append((a - hi.float()).clamp(-65504, 65504).half())
    return torch.stack(out).view(torch.int16)


def to_tf32(t, how):
    """fp32 -> tf32 (10-bit mantissa) by truncation, round-to-nearest-even or round-to-nearest-away."""
    i = t.contiguous().view(torch.int32)
    if how == "rne":
        i = i + 0xFFF + ((i >> 13) & 1)
    elif how == "rna":
        i = i + 0x1000
    return (i & ~0x1FFF).view(torch.float32)


def f16_operands(x, w):
    """The hi planes the f16 family multiplies, back in fp32: x at the activation scale 16, w at the layer's
    power-of-two scale (weight_scale: s * max|w| in [2^13, 2^14))."""
    xh = (x * 16).clamp(-65504, 65504).half().float() / 16
    m = float(w.abs().max())
    k = 0 if not (m > 0 and math.isfinite(m)) else max(-60, min(60, 14 - math.frexp(m)[1]))
    s = 2.0 ** k
    return xh, (w * s).clamp(-65504, 65504).half().float() / s


def reference(x, w, bias, act, resid, lens):
    """float64 conv1d ("same" padding per utterance) as a sum of shifted matmuls, + bias, act, + residual, zeros past lens."""
    taps, L = w.shape[0], x.shape[1]
    pad = (taps - 1) // 2
    xp = F.pad(x.double(), (0, 0, pad, pad))
    y = sum(xp[:, j:j + L] @ w[j].double().T for j in range(taps))
    if bias is not None:
        y = y + bias.double()
    y = torch.relu(y) if act == 1 else torch.tanh(y) if act == 2 else y
    if resid is not None:
        y = y + resid.double()
    if lens is not None:
        y = y.masked_fill(~valid_rows(lens, L)[..., None], 0.0)
    return y


def valid_rows(lens, L):
    return torch.arange(L, device=lens.device)[None, :] < lens[:, None]


def gates(fam, x, w):
    """(label, x, w, max gate, mean gate): the operands each gate compares against."""
    if fam == "fp32":
        return [("exact", x, w, 2e-5, 2e-6)]
    if fam == "3xf16":
        return [("exact", x, w, 5e-4, 5e-5)]
    if fam == "f16":
        return [("fp16 operands", *f16_operands(x, w), 5e-4, 5e-5), ("exact", x, w, 1e-2, 1e-3)]
    return [(f"tf32 operands ({TF32_CONVERSION})", to_tf32(x, TF32_CONVERSION), to_tf32(w, TF32_CONVERSION), 5e-4, 5e-5),
            ("exact", x, w, 1e-2, 1e-3)]


def check_numbers(fam, c, d, got):
    """got against float64 on the rows t < lens[b]; each case prints its max / mean error per gate."""
    mask = valid_rows(d["lens"], c.L) if d["lens"] is not None else torch.ones(c.B, c.L, dtype=torch.bool, device=DEV)
    for label, xx, ww, gmax, gmean in gates(fam, d["x"], d["w"]):
        want = reference(xx, ww, d["bias"], c.act, d["resid"], d["lens"])
        err = (got.double() - want)[mask].abs()
        mx, mn = (float(err.max()), float(err.mean())) if err.numel() else (0.0, 0.0)
        gmax, gmean = gmax * c.wscale, gmean * c.wscale
        print(f"GATE {fam:6s} {c.name:26s} {label:24s} max {mx:.3e} / {gmax:.1e}  mean {mn:.3e} / {gmean:.1e}")
        assert mx <= gmax and mn <= gmean, (fam, c.name, label, mx, mn)


_DATA = {}


def case_data(c):
    """Seeded inputs of a case (the same in every family); x holds zeros at rows t >= lens[b]."""
    if c.name not in _DATA:
        g = torch.Generator(device=DEV).manual_seed(zlib.crc32(c.name.encode()))
        x = torch.randn(c.B, c.L, c.K, generator=g, device=DEV)
        w = torch.randn(c.taps, c.N, c.K, generator=g, device=DEV) * (c.wscale / math.sqrt(c.K * c.taps))
        bias = torch.randn(c.N, generator=g, device=DEV) * c.wscale if c.bias else None
        resid = torch.randn(c.B, c.L, c.N, generator=g, device=DEV) * c.wscale if c.resid else None
        lens = torch.tensor(c.lens, dtype=torch.int64, device=DEV) if c.lens is not None else None
        if lens is not None:
            x = x.masked_fill(~valid_rows(lens, c.L)[..., None], 0.0)
        _DATA[c.name] = dict(x=x, w=w, bias=bias, resid=resid, lens=lens)
    return _DATA[c.name]


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module", autouse=True)
def _free_case_data():
    yield
    _DATA.clear()


def _ids(cases):
    return [c.name for c in cases]


# ---- GPU tests -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_is_covered_by_the_case_table(sms):
    assert check_coverage(sms) == [], f"the case table does not cover a {sms}-SM device"


@pytest.mark.gpu
def test_tf32_operand_conversion():
    """Which conversion the tf32 wgmma applies to fp32 operands in shared memory.  Each probe sits in the bits below the
    tf32 mantissa, so truncation, round-to-nearest-even and round-to-nearest-away give different products with 1.0;
    one call puts the probes in A (x), one in B (w).  Observed on an H100 SXM: truncation, in both operands."""
    e = [2.0 ** -11, 3 * 2.0 ** -12, 2.0 ** -10 + 2.0 ** -11, 2.0 ** -12, 2.0 ** -11 + 2.0 ** -13]
    probes = torch.tensor([s * (1.0 + d) for d in e for s in (1.0, -1.0)] + [1.5 + 2.0 ** -11] * 6, device=DEV)
    assert probes.numel() == 16
    eye = torch.eye(16, 32, device=DEV)
    x = torch.zeros(1, 1, 32, device=DEV)
    x[0, 0, :16] = probes
    got_a = tap_gemm("tf32", x, eye[None].contiguous(), None, 0, None)[0].flatten()
    ones = torch.zeros(1, 1, 32, device=DEV)
    ones[0, 0, :16] = 1.0
    got_b = tap_gemm("tf32", ones, (eye * probes[:, None])[None].contiguous(), None, 0, None)[0].flatten()
    seen = [how for how in ("truncate", "rne", "rna") if torch.equal(got_a, to_tf32(probes, how))]
    seen_b = [how for how in ("truncate", "rne", "rna") if torch.equal(got_b, to_tf32(probes, how))]
    print(f"tf32 operand conversion observed: A {seen}, B {seen_b}")
    assert seen == [TF32_CONVERSION] and seen_b == [TF32_CONVERSION], (got_a.tolist(), got_b.tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("fam,c", [(fam, c) for fam in FAMILIES for c in SCHEDULE_CASES[fam]],
                         ids=[c.name for fam in FAMILIES for c in SCHEDULE_CASES[fam]])
def test_schedule_cases_vs_float64(fam, c):
    """Every instantiation at every tile count and ring depth that matters: numbers against float64, and in the plane
    families the operand planes bit for bit against split_pair of the fp32 output."""
    d = case_data(c)
    planes = fam in PLANES
    out, pl, _ = tap_gemm(fam, d["x"], d["w"], d["bias"], c.act, d["resid"], planes=planes)
    check_numbers(fam, c, d, out)
    if planes:
        assert torch.equal(pl.view(torch.int16), split_planes(out.reshape(-1, c.N), PLANES[fam]))


@pytest.mark.gpu
@pytest.mark.parametrize("fam", FAMILIES)
@pytest.mark.parametrize("c", PER_UTT_CASES, ids=_ids(PER_UTT_CASES))
def test_per_utterance_contract(fam, c):
    """lens: numbers against float64; rows t >= lens[b] exactly +0 in out and every plane (dead tiles included); each
    utterance bit-identical to a B = 1 call of its own length and to the batch reversed; planes equal with and without
    the fp32 output; for plain GEMMs, NaN in the padded rows of x and of the residual changes nothing."""
    d = case_data(c)
    x, w, bias, resid, lens = d["x"], d["w"], d["bias"], d["resid"], d["lens"]
    planes = fam in PLANES
    P = PLANES.get(fam, 1)
    out, pl, _ = tap_gemm(fam, x, w, bias, c.act, resid, lens, planes=planes)
    check_numbers(fam, c, d, out)
    pad = ~valid_rows(lens, c.L)
    assert bool((bits(out)[pad] == 0).all()), "rows past lens are not +0"
    if planes:
        assert bool((bits(pl).view(P, c.B, c.L, c.N)[:, pad] == 0).all()), "plane rows past lens are not +0"
        assert torch.equal(bits(pl), split_planes(out.reshape(-1, c.N), P))
        assert torch.equal(bits(tap_gemm(fam, x, w, bias, c.act, resid, lens, out=False, planes=True)[1]), bits(pl))

    flip = [t.flip(0) if t is not None else None for t in (x, resid, lens)]
    out_r, pl_r, _ = tap_gemm(fam, flip[0], w, bias, c.act, flip[1], flip[2], planes=planes)
    assert torch.equal(bits(out_r.flip(0)), bits(out)), "reversing the batch changed the result"
    if planes:
        assert torch.equal(bits(pl_r).view(P, c.B, c.L, c.N).flip(1), bits(pl).view(P, c.B, c.L, c.N))

    for b, n in enumerate(c.lens):
        if n == 0:
            continue
        o1, p1, _ = tap_gemm(fam, x[b:b + 1, :n].contiguous(), w, bias, c.act,
                             resid[b:b + 1, :n].contiguous() if resid is not None else None, planes=planes)
        assert torch.equal(bits(o1[0]), bits(out[b, :n])), f"utterance {b} differs from its B = 1 run"
        if planes:
            assert torch.equal(bits(p1), bits(pl).view(P, c.B, c.L, c.N)[:, b, :n])

    if c.taps == 1:
        xn = x.masked_fill(pad[..., None], float("nan"))
        rn = resid.masked_fill(pad[..., None], float("nan")) if resid is not None else None
        out_n, pl_n, _ = tap_gemm(fam, xn, w, bias, c.act, rn, lens, planes=planes)
        assert torch.equal(bits(out_n), bits(out)), "NaN in padded rows reached the output"
        if planes:
            assert torch.equal(bits(pl_n), bits(pl))


@pytest.mark.gpu
@pytest.mark.parametrize("fam", TC_FAMILIES)
@pytest.mark.parametrize("c", VT_CASES, ids=_ids(VT_CASES))
def test_transposed_v(fam, c):
    """q|k|v projection with the V third stored transposed: Vᵀ (and its planes) bit for bit against the plain call's V
    columns, itself checked against float64; q|k columns unchanged; out and out_planes untouched in the V columns;
    Vᵀ entries at t >= lens[b] and t in [L, lpad) never written; plain GEMM rows past lens hold NaN in x."""
    d = case_data(c)
    x, w, bias, lens = d["x"], d["w"], d["bias"], d["lens"]
    planes = fam in PLANES
    P = PLANES.get(fam, 1)
    col0, lpad = 2 * c.N // 3, lpad_of(c.L)
    dk = (c.N - col0) // VT_HEADS
    ref_out, ref_pl, _ = tap_gemm(fam, x, w, bias, c.act, None, lens, planes=planes)
    check_numbers(fam, c, d, ref_out)
    xn = x.masked_fill(~valid_rows(lens, c.L)[..., None], float("nan")) if lens is not None else x
    out, pl, vt = tap_gemm(fam, xn, w, bias, c.act, None, lens, planes=planes, vt=(col0, VT_HEADS, lpad))

    assert torch.equal(bits(out[..., :col0]), bits(ref_out[..., :col0]))
    assert bool((bits(out[..., col0:]) == SENT32).all()), "out was written in the V columns"
    n_valid = lens if lens is not None else torch.full((c.B,), c.L, device=DEV)
    written = (torch.arange(lpad, device=DEV)[None, :] < n_valid[:, None]).repeat_interleave(VT_HEADS, 0)[:, None, :]
    v = ref_out[..., col0:].reshape(c.B, c.L, VT_HEADS, dk).permute(0, 2, 3, 1).reshape(c.B * VT_HEADS, dk, c.L)
    v = F.pad(v, (0, lpad - c.L))
    if fam == "tf32":
        want = torch.where(written, bits(v), torch.full_like(bits(v), SENT32))
        assert torch.equal(bits(vt), want), "transposed V"
    else:
        sp = split_planes(v, P)
        want = torch.where(written[None], sp, torch.full_like(sp, SENT16))
        assert torch.equal(bits(vt), want), "transposed V planes"
        plv = bits(pl).view(P, c.B * c.L, c.N)
        assert torch.equal(plv[..., :col0], bits(ref_pl)[..., :col0])
        assert bool((plv[..., col0:] == SENT16).all()), "out_planes was written in the V columns"
        vt_only = tap_gemm(fam, xn, w, bias, c.act, None, lens, out=False, vt=(col0, VT_HEADS, lpad))[2]
        assert torch.equal(bits(vt_only), bits(vt))


@pytest.mark.gpu
@pytest.mark.parametrize("fam", TC_FAMILIES)
@pytest.mark.parametrize("c", INDEPENDENCE_CASES, ids=_ids(INDEPENDENCE_CASES))
def test_schedule_independence(fam, c, sms):
    """Each utterance alone (every CTA one tile, warpgroup 0 only) and inside a batch of more than 2 x SMs tiles, where
    some of its tiles run on warpgroup 1 after a carried-over ring: the same bits, out and planes."""
    t = c.tiling()
    assert tiling(1, c.L, c.N, c.taps, False).total <= sms and t.total > 2 * sms
    assert any(len(cta) > 1 for cta in walk(t, None, sms)), "no tile of the batch runs on warpgroup 1"
    d = case_data(c)
    planes = fam in PLANES
    P = PLANES.get(fam, 1)
    out, pl, _ = tap_gemm(fam, d["x"], d["w"], d["bias"], c.act, d["resid"], planes=planes)
    check_numbers(fam, c, d, out)
    for b in range(c.B):
        o1, p1, _ = tap_gemm(fam, d["x"][b:b + 1].contiguous(), d["w"], d["bias"], c.act,
                             d["resid"][b:b + 1].contiguous() if d["resid"] is not None else None, planes=planes)
        assert torch.equal(bits(o1[0]), bits(out[b])), f"utterance {b}: batch and alone differ"
        if planes:
            assert torch.equal(bits(p1), bits(pl).view(P, c.B, c.L, c.N)[:, b])
