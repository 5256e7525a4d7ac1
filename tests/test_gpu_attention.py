"""The self-attention kernels against float64: attention_tc.cu's attention_wgmma_kernel (f16, 3xf16) through
fs2_op_attention_planes, on q|k and Vᵀ operand planes this file writes byte for byte, and attention_tc_kernel (tf32) and
attention_fp32.cu (fp32) through fs2_op_attention.

The wgmma kernel runs one CTA per 128 queries of one (batch, head): a TMA producer warp and two consumer warpgroups of
64 rows, `active` of them with a row below len, and a ring of STAGES K / Vᵀ slots that every CTA walks over the
ceil(len / 64) key tiles of its utterance.  The producer zeroes the Vᵀ columns >= len of a partial last key tile in
shared memory.  This file restates the ring depth in Python and chooses its cases with it.  The CPU tests assert what
the case table reaches for each of the four instantiations (d_k 128 / 192, f16 / 3xf16); the GPU tests check:

  * every case in every family against a float64 masked softmax, with exact-operand gates, and in f16 / tf32 a tight
    gate against float64 on the operands as the kernel rounds them;
  * NaN in every q|k row and Vᵀ column the kernel must not read for its values (t >= len, and Vᵀ in [L, lpad)): the
    valid rows keep their bits, rows past len are +0 in ctx and in every context plane;
  * the context planes bit for bit against split_pair of ctx, with and without ctx;
  * an utterance alone and inside a ragged batch (and the reversed batch) with NaN padding: the same bits;
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
from test_gpu_tap_gemm import DEV, SENT16, SENT32, Guarded, bits, split_planes, to_tf32

# ---- restatement of the wgmma kernel's configuration (attention_tc.cu, FCfg) ----------------------------------------
FA_BQ, FA_BKV = 128, 64                      # queries per CTA (two consumer warpgroups of 64), keys per tile
BUDGET = 227 * 1024 - 1024 - 256             # shared memory: 227 KB less alignment slack and barriers
PLANE_FAMILIES = ("f16", "3xf16")            # attention_wgmma_kernel<DK, X3 = false / true>
FAMILIES = ("fp32", "tf32") + PLANE_FAMILIES
MODE = {"fp32": _lib.MATH_FP32, "tf32": _lib.MATH_TF32, "f16": _lib.MATH_F16, "3xf16": _lib.MATH_3XTF32}
PLANES = {"f16": 1, "3xf16": 2}
DKS = (128, 192)
INSTANTIATIONS = [(dk, fam) for dk in DKS for fam in PLANE_FAMILIES]
NAN16 = 0x7E00


def fcfg(dk, fam):
    """FCfg<DK, X3>: (Q bytes, bytes per ring stage, STAGES).  Q is [plane][d_k / 64 swizzle atoms][128 rows][128 B];
    a stage is one K box [plane][atom][64 keys][128 B] and one Vᵀ box [plane][d_k rows][64 keys x 2 B]; at most 2."""
    P, atoms = PLANES[fam], dk // 64
    q_bytes = P * atoms * FA_BQ * 128
    stage = P * atoms * FA_BKV * 128 + P * dk * 128
    return q_bytes, stage, min(2, (BUDGET - q_bytes) // stage)


def stages(dk, fam):
    return fcfg(dk, fam)[2]


def key_tiles(n):
    return -(-n // FA_BKV)


def active(n, q0):
    """Consumer warpgroups of the CTA at q0 with a row below len n."""
    return 0 if q0 >= n else 1 if q0 + 64 >= n else 2


def round8(n):
    return (n + 7) // 8 * 8


# ---- cases -------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Case:
    name: str
    B: int
    L: int
    C: int
    heads: int
    lens: Optional[Tuple[int, ...]] = None   # None: unmasked (lens = NULL)
    lpad_extra: int = 0                      # Vᵀ row pitch round8(L) + this
    kind: str = "randn"                      # randn | peaked | underflow | mean (see make_inputs)

    @property
    def dk(self):
        return self.C // self.heads

    @property
    def lpad(self):
        return round8(self.L) + self.lpad_extra

    @property
    def n(self):
        """Keys (and output rows) of each utterance."""
        return self.lens if self.lens is not None else (self.L,) * self.B

    @property
    def sstd(self):
        """Standard deviation of the scores: the exact-operand gates scale with it."""
        return 10.0 if self.kind == "peaked" else 1.0


# len mod 128 around the 16 / 32 / 64 boundaries (L = 256) and a batch of more CTAs than SMs with lens 0, 1, L and
# ends inside a key tile (L = 1000)
PARTIAL_LENS = tuple(128 + r for r in (1, 15, 16, 17, 31, 32, 33, 48, 63, 64, 65, 96, 112, 127, 128))
WAVES_LENS = (1000, 0, 999, 130, 128, 1, 517, 1000, 64, 900, 0, 385, 1000, 257)
RESIDUE_LENS = tuple(r + 64 * (r % 5) for r in range(64))      # every len mod 64, 1 to 5 key tiles


def _cases(dk):
    return [
        Case(f"partial-dk{dk}", 15, 256, 2 * dk, 2, PARTIAL_LENS),
        Case(f"waves-dk{dk}", 14, 1000, 2 * dk, 2, WAVES_LENS),
        Case(f"residues-h3-dk{dk}", 64, 321, 3 * dk, 3, RESIDUE_LENS, lpad_extra=8),
        Case(f"short-h1-dk{dk}", 4, 40, dk, 1, (40, 1, 23, 0), lpad_extra=16),
        Case(f"unmasked-L145-dk{dk}", 2, 145, 2 * dk, 2),
        Case(f"unmasked-L168-dk{dk}", 2, 168, 2 * dk, 2, lpad_extra=8),
        Case(f"unmasked-L385-dk{dk}", 2, 385, 2 * dk, 2),
        Case(f"unmasked-h1-L40-dk{dk}", 2, 40, dk, 1, lpad_extra=8),
        Case(f"unmasked-h3-L200-dk{dk}", 1, 200, 3 * dk, 3),
        Case(f"peaked-dk{dk}", 3, 300, 2 * dk, 2, (300, 237, 75), kind="peaked"),
        Case(f"underflow-h1-dk{dk}", 2, 260, dk, 1, (260, 200), kind="underflow"),
        Case(f"mean-h3-dk{dk}", 3, 150, 3 * dk, 3, (150, 129, 64), kind="mean"),
    ]


CASES = [c for dk in DKS for c in _cases(dk)]
INDEPENDENCE_CASES = [c for c in CASES if c.name.startswith(("partial", "waves"))]


# ---- what the table covers -----------------------------------------------------------------------------------------
ACTIVE_BOUNDARIES = {0: 0, 1: 1, 64: 1, 65: 2, 128: 2}       # len - q0 -> active warpgroups of the CTA at q0


def coverage(dk, fam):
    S = stages(dk, fam)
    facts = set()
    for c in (c for c in CASES if c.dk == dk):
        for n in c.n:
            t = key_tiles(n)
            facts |= {f"{what} key tiles" for what, k in (("1", 1), ("S", S), ("S + 1", S + 1)) if t == k}
            if t >= 4 * S + 1:
                facts.add(">= 4 S + 1 key tiles")
            facts.add(f"len % 64 = {n % 64}")
            for q0 in range(FA_BQ, c.L, FA_BQ):
                if n - q0 in ACTIVE_BOUNDARIES:
                    facts.add(f"len = q0 + {n - q0}, active {active(n, q0)}")
            if n % FA_BQ and n > c.L // FA_BQ * FA_BQ:
                facts.add("Q box crosses L")
            if n == 0:
                facts.add("len 0")
        if c.L < 64:
            facts.add("L < 64")
        if c.L % FA_BQ:
            facts.add("L % 128 != 0")
        if c.lpad > round8(c.L):
            facts.add("lpad > round8(L)")
        if c.lens is None and c.L % FA_BKV and c.lpad > c.L:
            facts.add("unmasked, last key tile reads Vᵀ in [L, lpad)")
        facts.add(f"heads {c.heads}")
        facts.add(f"kind {c.kind}")
    return facts


def wanted(dk, fam):
    want = {"1 key tiles", "S key tiles", "S + 1 key tiles", ">= 4 S + 1 key tiles", "Q box crosses L", "len 0",
            "L < 64", "L % 128 != 0", "lpad > round8(L)", "unmasked, last key tile reads Vᵀ in [L, lpad)",
            "heads 1", "heads 2", "heads 3", "kind randn", "kind peaked", "kind underflow", "kind mean"}
    want |= {f"len % 64 = {r}" for r in range(64)}
    want |= {f"len = q0 + {d}, active {a}" for d, a in ACTIVE_BOUNDARIES.items()}
    return want


def check_coverage():
    missing = [(dk, fam, f) for dk, fam in INSTANTIATIONS for f in sorted(wanted(dk, fam) - coverage(dk, fam))]
    for c in CASES:
        if c.dk not in DKS or c.C % c.heads or (c.B * c.L * c.C) % 16 or (c.lens and max(c.lens) > c.L):
            missing.append((c.name, "shape"))
    for c in INDEPENDENCE_CASES:
        if c.lens is None or len(set(c.lens)) < 3:
            missing.append((c.name, "independence needs a ragged batch"))
    return missing


def test_case_table_covers_the_kernel():
    """For each instantiation: 1, S, S + 1 and >= 4 S + 1 key tiles, every len mod 64, CTAs with 0 / 1 / 2 active
    warpgroups at len = q0, q0 + 1, q0 + 64, q0 + 65, q0 + 128, L < 64, L % 128 != 0, lpad > round8(L), heads 1-3."""
    assert check_coverage() == []


def test_ring_depth_restatement():
    """STAGES is 1 for <192, 3xf16> (Q 96 KB, one stage 96 KB) and 2 for the other three; everything fits in 227 KB."""
    assert {(dk, fam): stages(dk, fam) for dk, fam in INSTANTIATIONS} == {
        (128, "f16"): 2, (128, "3xf16"): 2, (192, "f16"): 2, (192, "3xf16"): 1}
    assert fcfg(192, "3xf16")[:2] == (96 * 1024, 96 * 1024)
    for dk, fam in INSTANTIATIONS:
        q_bytes, stage, S = fcfg(dk, fam)
        assert q_bytes + S * stage + 1024 + 256 <= 227 * 1024


def test_rejects_bad_arguments_on_the_host():
    """Both entries refuse these before they touch memory (the pointers are never dereferenced)."""
    lib = _lib.load()
    p = 256     # a stand-in non-null, aligned pointer

    def planes(mode=_lib.MATH_3XTF32, qkp=p, vtp=p, lpad=264, L=257, ctx=p, ctxp=None):
        return lib.fs2_op_attention_planes(mode, qkp, vtp, lpad, None, 2, L, 384, 2, ctx, ctxp, None)

    for mode in (_lib.MATH_FP32, _lib.MATH_TF32, 7, -1):
        assert planes(mode=mode) == -1 and b"math mode" in lib.fs2_last_error()
    for mode in (7, -1):
        assert lib.fs2_op_attention(mode, p, None, 2, 257, 384, 2, p, None) == -1 and b"math mode" in lib.fs2_last_error()
    assert planes(ctx=None) == -1 and b"no output" in lib.fs2_last_error()
    assert planes(lpad=256) == -1 and b"row pitch" in lib.fs2_last_error()          # lpad < L
    assert planes(lpad=260) == -1 and b"row pitch" in lib.fs2_last_error()          # lpad % 8 != 0
    assert planes(qkp=p + 8) == -1 and b"16-byte aligned" in lib.fs2_last_error()
    assert planes(vtp=p + 2) == -1 and b"16-byte aligned" in lib.fs2_last_error()
    assert planes(ctxp=p + 16) == -1 and b"32-byte aligned" in lib.fs2_last_error()
    assert planes(mode=_lib.MATH_F16, vtp=None) == -1


# ---- inputs --------------------------------------------------------------------------------------------------------
def make_inputs(c):
    """Seeded q, k, v [B, L, C] fp32 on the CPU, zeros at rows t >= len (the production state: every GEMM family writes
    them so).  randn: N(0, 1).  peaked: scores of std ~10 (q x 10), and in each head the channel-0 pair q = 16,
    k = round(2.5 sqrt(d_k)) on the keys of the last (partial) key tile lifts those scores by ~40, so every valid row
    takes its maximum there and the running maximum rescales all earlier tiles by corr << 1.  underflow: k = -round(14.5
    sqrt(d_k)) in channel 0 on the keys of tile 1 puts its scores ~200 below the running maximum of tile 0, so the whole
    tile underflows to 0.  mean: q = 0, so each valid row is the mean of V over the valid keys.  The channel-0 values
    are exact in the fp16 planes."""
    g = torch.Generator().manual_seed(zlib.crc32(c.name.encode()))
    q, k, v = (torch.randn(c.B, c.L, c.C, generator=g) for _ in range(3))
    dk, ch0 = c.dk, slice(0, c.C, c.dk)
    if c.kind == "peaked":
        q *= 10.0
        q[..., ch0] = 16.0
        k[..., ch0] = 0.0
        for b, n in enumerate(c.n):
            k[b, (n - 1) // FA_BKV * FA_BKV:n, ch0] = float(round(2.5 * math.sqrt(dk)))
    elif c.kind == "underflow":
        q[..., ch0] = 16.0
        k[..., ch0] = 0.0
        k[:, FA_BKV:2 * FA_BKV, ch0] = -float(round(14.5 * math.sqrt(dk)))
    elif c.kind == "mean":
        q.zero_()
    if c.lens is not None:
        past = torch.arange(c.L)[None, :] >= torch.tensor(c.lens)[:, None]
        for t in (q, k, v):
            t[past] = 0.0
    return q, k, v


def scores(q, k, heads):
    B, L, C = q.shape
    dk = C // heads
    qh, kh = (t.double().view(B, L, heads, dk).transpose(1, 2) for t in (q, k))
    return qh @ kh.transpose(-1, -2) / math.sqrt(dk)


def key_mask(n, L, device):
    return torch.arange(L, device=device)[None, :] < torch.as_tensor(n, device=device)[:, None]


def reference(q, k, v, n, heads):
    """float64: softmax over the keys u < n[b], P.V, exact zeros at rows t >= n[b] (and for n[b] = 0)."""
    B, L, C = q.shape
    valid = key_mask(n, L, q.device)
    s = scores(q, k, heads).masked_fill(~valid[:, None, None, :], -math.inf)
    p = torch.softmax(s, -1).nan_to_num(0.0)
    o = (p @ v.double().view(B, L, heads, C // heads).transpose(1, 2)).transpose(1, 2).reshape(B, L, C)
    return o.masked_fill(~valid[..., None], 0.0)


def test_special_inputs_do_what_they_claim():
    """peaked: score std 8-12, every valid row's maximum in the last key tile; underflow: tile 1 at least 150 below
    every row's maximum over tile 0 (exp underflows to 0 in fp32); mean: q = 0."""
    for c in CASES:
        if c.kind == "randn":
            continue
        q, k, v = make_inputs(c)
        s = scores(q, k, c.heads)
        for b, n in enumerate(c.n):
            sb = s[b, :, :n, :n]
            if c.kind == "peaked":
                last = (n - 1) // FA_BKV * FA_BKV
                assert n % FA_BKV and bool((sb.argmax(-1) >= last).all()), (c.name, b)
                assert 8 < float(sb[..., :last].std()) < 12, c.name
            elif c.kind == "underflow":
                assert n > 2 * FA_BKV
                assert bool((sb[..., FA_BKV:2 * FA_BKV].amax(-1) < sb[..., :FA_BKV].amax(-1) - 150).all()), c.name
            else:
                assert bool((q == 0).all())


# ---- GPU: operands and calls ----------------------------------------------------------------------------------------
_DATA, _REF = {}, {}


def case_data(c):
    if c.name not in _DATA:
        q, k, v = (t.to(DEV) for t in make_inputs(c))
        lens = torch.tensor(c.lens, dtype=torch.int64, device=DEV) if c.lens is not None else None
        _DATA[c.name] = dict(q=q, k=k, v=v, lens=lens)
    return _DATA[c.name]


def plane_operands(q, k, v, n, heads, lpad, P, nan):
    """q|k planes [P][B*L][2C] and Vᵀ planes [P][B*heads][d_k][lpad] as the projection's epilogue writes them
    (split_pair of 16 x); nan: fp16 NaN in every q|k row and Vᵀ column at t >= n[b], and in the Vᵀ columns [L, lpad)."""
    B, L, C = q.shape
    qkp = split_planes(torch.cat([q, k], -1), P)                                   # [P, B, L, 2C]
    vt = F.pad(v.view(B, L, heads, C // heads).permute(0, 2, 3, 1), (0, lpad - L))  # [B, heads, d_k, lpad]
    vtp = split_planes(vt, P)
    if nan:
        nan16 = torch.tensor(NAN16, dtype=torch.int16, device=q.device)
        qkp = torch.where(~key_mask(n, L, q.device)[None, :, :, None], nan16, qkp)
        vtp = torch.where(~key_mask(n, lpad, q.device)[None, :, None, None, :], nan16, vtp)
    return (qkp.reshape(P, B * L, 2 * C).contiguous().view(torch.float16),
            vtp.reshape(P, B * heads, C // heads, lpad).contiguous().view(torch.float16))


def attention(fam, q, k, v, lens, heads, lpad, *, nan=False, ctx=True, ctxp=False):
    """One call on sentinel-guarded outputs: ctx [B, L, C] and the context planes [P, B*L, C] (None when not asked for).
    nan: NaN past the lengths -- in the plane families everywhere plane_operands puts it; in fp32 / tf32 in the k and v
    thirds only (those kernels read q rows below L and scale the rows past len by 0, so q stays 0 there)."""
    lib = _lib.load()
    B, L, C = q.shape
    n = lens if lens is not None else torch.full((B,), L, device=q.device)
    rows = B * L
    g_ctx = Guarded(rows * C, torch.float32) if ctx else None
    g_pl = None
    if fam in PLANES:
        P = PLANES[fam]
        # f16 writes the hi plane only: the band after it is as large as a lo plane would be
        g_pl = Guarded(P * rows * C, torch.float16, post=rows * C if P == 1 else 0) if ctxp else None
        qkp, vtp = plane_operands(q, k, v, n, heads, lpad, P, nan)
        rc = lib.fs2_op_attention_planes(MODE[fam], _lib.ptr(qkp), _lib.ptr(vtp), lpad, _lib.ptr(lens), B, L, C, heads,
                                         _lib.ptr(g_ctx.view) if ctx else None, _lib.ptr(g_pl.view) if ctxp else None,
                                         _lib.stream_ptr(q.device))
        _lib.check(rc, "fs2_op_attention_planes")
    else:
        assert ctx and not ctxp
        if nan:
            past = ~key_mask(n, L, q.device)[..., None]
            k, v = k.masked_fill(past, float("nan")), v.masked_fill(past, float("nan"))
        qkv = torch.cat([q, k, v], -1).contiguous()
        rc = lib.fs2_op_attention(MODE[fam], _lib.ptr(qkv), _lib.ptr(lens), B, L, C, heads, _lib.ptr(g_ctx.view),
                                  _lib.stream_ptr(q.device))
        _lib.check(rc, "fs2_op_attention")
    torch.cuda.synchronize()
    for name, g in (("ctx", g_ctx), ("ctxp", g_pl)):
        assert g is None or g.intact(), f"{fam}: a store landed outside {name}"
    return (g_ctx.view.view(B, L, C) if ctx else None, g_pl.view.view(-1, rows, C) if ctxp else None)


def run_case(fam, c, **kw):
    d = case_data(c)
    return attention(fam, d["q"], d["k"], d["v"], d["lens"], c.heads, c.lpad, **kw)


def f16_operand(t):
    """What the hi plane holds, back in fp32: rn_fp16(sat(16 t)) / 16."""
    return split_planes(t, 1)[0].view(torch.float16).float() / 16


# Tight gates (max, mean) against the rounded operands, about 4x / 7x the worst case over the table measured on an
# NVIDIA H100 80GB HBM3 at a 400 W power limit (the GATE lines this file prints): f16 max 4.9e-4 (peaked-dk128), mean
# 3.0e-5 (short-h1-dk192); tf32 max 5.6e-4 (peaked-dk192), mean 3.1e-5 (short-h1-dk192).  The exact-operand error of
# the same cases is 2-30x larger.
TIGHT = {"f16": (2e-3, 2e-4), "tf32": (2e-3, 2e-4)}


def gates(fam):
    """(label, operand map, max gate, mean gate, scales with the score std)."""
    if fam == "fp32":
        return [("exact", None, 2e-5, 2e-6, True)]
    if fam == "3xf16":
        return [("exact", None, 5e-5, 5e-6, True)]
    rounded = ("fp16 operands", f16_operand) if fam == "f16" else ("tf32 operands (rna)", lambda t: to_tf32(t, "rna"))
    return [(*rounded, *TIGHT[fam], False), ("exact", None, 1e-2, 1e-3, True)]


def want(c, label, fn):
    key = (c.name, label)
    if key not in _REF:
        d = case_data(c)
        q, k, v = (fn(t) if fn else t for t in (d["q"], d["k"], d["v"]))
        _REF[key] = reference(q, k, v, c.n, c.heads)
    return _REF[key]


@pytest.fixture(scope="module", autouse=True)
def _free_case_data():
    yield
    _DATA.clear()
    _REF.clear()


def _ids(cases):
    return [c.name for c in cases]


# ---- GPU tests -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fam", FAMILIES)
@pytest.mark.parametrize("c", CASES, ids=_ids(CASES))
def test_vs_float64(fam, c):
    """Valid rows against float64 per gate (each case prints its max / mean error); rows past len are 0 (+0 bits in the
    plane families, where the epilogue selects 0; o x 0 of either sign in fp32 / tf32)."""
    got, _ = run_case(fam, c)
    valid = key_mask(c.n, c.L, DEV)
    for label, fn, gmax, gmean, scales in gates(fam):
        err = (got.double() - want(c, label, fn))[valid].abs()
        mx, mn = (float(err.max()), float(err.mean())) if err.numel() else (0.0, 0.0)
        if scales:
            gmax, gmean = gmax * c.sstd, gmean * c.sstd
        print(f"GATE {fam:5s} {c.name:26s} {label:20s} max {mx:.3e} / {gmax:.1e}  mean {mn:.3e} / {gmean:.1e}")
        assert mx <= gmax and mn <= gmean, (fam, c.name, label, mx, mn)
    if fam in PLANES:
        assert bool((bits(got)[~valid] == 0).all()), "rows past len are not +0"
    else:
        assert bool((got[~valid] == 0).all()), "rows past len are not 0"


@pytest.mark.gpu
@pytest.mark.parametrize("fam", FAMILIES)
@pytest.mark.parametrize("c", CASES, ids=_ids(CASES))
def test_nan_past_the_lengths(fam, c):
    """NaN in every operand the kernel must not read for its values gives the bits of the zero-padded call (in the plane
    families that includes Vᵀ columns [L, lpad) of unmasked calls, which the last key tile's box reads)."""
    if fam not in PLANES and c.lens is None:
        pytest.skip("fp32 / tf32 without lens: no row past len")
    ref, _ = run_case(fam, c)
    got, _ = run_case(fam, c, nan=True)
    valid = key_mask(c.n, c.L, DEV)
    assert torch.equal(bits(got)[valid], bits(ref)[valid]), "NaN padding changed a valid row"
    if fam in PLANES:
        assert bool((bits(got)[~valid] == 0).all()), "rows past len are not +0"
    else:
        assert bool((got[~valid] == 0).all()), "rows past len are not 0"


@pytest.mark.gpu
@pytest.mark.parametrize("fam", PLANE_FAMILIES)
@pytest.mark.parametrize("c", CASES, ids=_ids(CASES))
def test_context_planes(fam, c):
    """The context planes (what the out-projection reads) equal split_pair of ctx bit for bit, with NaN padding; a
    ctxp-only call gives the same bits; rows past len are +0 in every plane; f16 leaves the lo-plane-sized band after
    the hi plane untouched (Guarded checks it)."""
    P = PLANES[fam]
    ctx, pl = run_case(fam, c, nan=True, ctxp=True)
    assert torch.equal(bits(pl), split_planes(ctx.reshape(-1, c.C), P))
    past = ~key_mask(c.n, c.L, DEV).reshape(-1)
    assert bool((bits(pl)[:, past] == 0).all())
    _, pl_only = run_case(fam, c, nan=True, ctx=False, ctxp=True)
    assert torch.equal(bits(pl_only), bits(pl))


@pytest.mark.gpu
@pytest.mark.parametrize("fam", FAMILIES)
@pytest.mark.parametrize("c", INDEPENDENCE_CASES, ids=_ids(INDEPENDENCE_CASES))
def test_utterance_alone_equals_its_rows_in_a_batch(fam, c):
    """DESIGN section 5: a row depends only on its utterance's len and its rows below len.  Each utterance alone (B = 1,
    L = len, lens = NULL, lpad = round8(len)) gives the bits of its rows inside the ragged batch at L = Lmax with NaN
    padding, and inside the reversed batch."""
    d = case_data(c)
    q, k, v, lens = d["q"], d["k"], d["v"], d["lens"]
    planes = fam in PLANES
    out, pl = attention(fam, q, k, v, lens, c.heads, c.lpad, nan=True, ctxp=planes)
    rev, pl_r = attention(fam, q.flip(0), k.flip(0), v.flip(0), lens.flip(0), c.heads, c.lpad, nan=True, ctxp=planes)
    rev = rev.flip(0)
    for b, n in enumerate(c.lens):
        if n == 0:
            continue
        u = [t[b:b + 1, :n].contiguous() for t in (q, k, v)]
        o1, p1 = attention(fam, *u, None, c.heads, round8(n), ctxp=planes)
        assert torch.equal(bits(o1[0]), bits(out[b, :n])), f"utterance {b}: alone and in the batch differ"
        assert torch.equal(bits(o1[0]), bits(rev[b, :n])), f"utterance {b}: alone and in the reversed batch differ"
        if planes:
            P = PLANES[fam]
            assert torch.equal(bits(p1), bits(pl).view(P, c.B, c.L, c.C)[:, b, :n])
            assert torch.equal(bits(p1), bits(pl_r).view(P, c.B, c.L, c.C)[:, c.B - 1 - b, :n])


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_fp32_attention_on_a_second_device():
    """The fp32 kernel's 163 KB of shared memory at d_k 192 needs the opt-in attribute on each device it runs on: run on
    cuda:0, then on cuda:1 in the same process."""
    c = Case("second-device", 2, 300, 384, 2, (300, 171))
    q, k, v = make_inputs(c)
    lib = _lib.load()
    for dev in (0, 1):
        with torch.cuda.device(dev):
            qkv = torch.cat([q, k, v], -1).to(f"cuda:{dev}")
            lens = torch.tensor(c.lens, dtype=torch.int64, device=f"cuda:{dev}")
            ctx = torch.full((c.B, c.L, c.C), float("nan"), device=f"cuda:{dev}")
            _lib.check(lib.fs2_op_attention(_lib.MATH_FP32, _lib.ptr(qkv), _lib.ptr(lens), c.B, c.L, c.C, c.heads,
                                            _lib.ptr(ctx), _lib.stream_ptr(ctx.device)), f"fs2_op_attention on cuda:{dev}")
            torch.cuda.synchronize()
            err = (ctx.double().cpu() - reference(q, k, v, c.n, c.heads)).abs()
            assert float(err.max()) <= 2e-5, (dev, float(err.max()))
