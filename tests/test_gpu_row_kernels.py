"""The row kernels of csrc/rowwise.cu against float64 and against the reference's integer rules, through
fs2_op_row_norm, fs2_op_layernorm, fs2_embed_posenc, fs2_op_variance_embed_add, fs2_bucketize and fs2_one_hot.

  a. LayerNorm against float64 on rows chosen to stress it (cancellation, outliers, variance below eps, constant rows);
  b. every fusion bit for bit with gamma = 0, where the LayerNorm gives beta exactly and the rest is fixed fp32
     arithmetic restated in numpy (tests/test_row_kernels_plan.py);
  c. the configurations the stages issue, with random gamma and beta, against float64;
  d. the duration rule at its ties, driven through the head;
  e. bucket edges, the variance gather and the one-hot;
  f. the encoder input embedding in its inference form;
  g. padding, per-utterance independence and launch geometry.

Gates are about 3x the worst value measured on an H100 (DESIGN.md section 4); each run prints `MEASURED name value`.
"""
import ctypes

import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib
from test_gpu_tap_gemm import PAD, SENT16, SENT32, Guarded, split_planes
from test_row_kernels_plan import (F32, TIE_KMAX, bin_sets, dur_truth, edge_values, exact_tie_candidates, exact_ties, fused_rows,
                                   special_set, tie_distance, tie_half_even, tie_set, uniform_set, variance_rows)

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENT64 = 0x7FA5A5A5A5A5A5A5
GATE = {"layernorm": 6e-7, "head": 7e-8}     # max |y - y64| / error scale (ln64, and the head's sum |y64 w| + |b|)
WORST = {}


def measured(name, value):
    WORST[name] = max(WORST.get(name, 0.0), value)
    print(f"MEASURED {name} {value:.3e}")


def bits(t):
    return t.contiguous().view({torch.float32: torch.int32, torch.float16: torch.int16, torch.int64: torch.int64}[t.dtype])


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


def rnd(shape, seed, scale=1.0, shift=0.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(shape, generator=g, device=DEV) * scale + shift


class Guarded64:
    """An int64 output between guard bands of sentinel values."""

    def __init__(self, n):
        self.n = n
        self.buf = torch.full((PAD + n + PAD,), SENT64, dtype=torch.int64, device=DEV)
        self.view = self.buf[PAD:PAD + n]

    def intact(self):
        return bool((self.buf[:PAD] == SENT64).all()) and bool((self.buf[PAD + self.n:] == SENT64).all())


def P(t):
    return None if t is None else _lib.ptr(t)


# ---- fs2_op_row_norm on guarded outputs -------------------------------------------------------------------------
def row_norm(x, gamma, beta, eps, *, rows=None, ldx=None, resid=None, ldr=None, out=True, ldo=None, relu=False, pe=None,
             alpha=None, L=0, head_w=None, head_b=None, head_out=False, dur_out=False, head_scale=None, lens=None, planes=0,
             spk_table=None, spk=None, spk_L=0):
    """One fs2_op_row_norm call.  planes: 0 none, 1 hi only (split_lo = 0), 2 hi + lo; the lo half is always allocated
    so that a hi-only call can be seen to leave it alone.  Returns a dict of out [rows, C], planes [2, rows, C] (fp16),
    head [rows], dur [rows], after checking every guard band and, with ldo > C, the columns past C."""
    Cn = gamma.numel()
    ldx = x.shape[-1] if ldx is None else ldx
    rows = x.numel() // max(ldx, 1) if rows is None else rows
    ldo = Cn if ldo is None else ldo
    g_out = Guarded(rows * ldo, torch.float32) if out else None
    g_pl = Guarded(2 * rows * Cn, torch.float16) if planes else None
    g_head = Guarded(rows, torch.float32) if head_out else None
    g_dur = Guarded64(rows) if dur_out else None
    d = _lib.RowNormDesc(x=P(x), ldx=ldx, resid=P(resid), ldr=ldr or 0, gamma=P(gamma), beta=P(beta), eps=eps, rows=rows, C=Cn,
                         out=P(g_out.view) if out else None, ldo=ldo, relu_after=int(relu), pe=P(pe), alpha=P(alpha), L=L,
                         head_w=P(head_w), head_b=P(head_b), head_out=P(g_head.view) if head_out else None,
                         dur_out=P(g_dur.view) if dur_out else None, head_scale=P(head_scale), lens=P(lens),
                         split_out=P(g_pl.view) if planes else None, split_lo=int(planes == 2), spk_table=P(spk_table),
                         spk=P(spk), n_spk=0 if spk_table is None else spk_table.shape[0], spk_L=spk_L)
    _lib.check(_lib.load().fs2_op_row_norm(ctypes.byref(d), _lib.stream_ptr(torch.device(DEV))), "fs2_op_row_norm")
    torch.cuda.synchronize()
    res = {}
    for name, g in (("out", g_out), ("planes", g_pl), ("head", g_head), ("dur", g_dur)):
        assert g is None or g.intact(), f"a store landed outside {name}"
    if out:
        full = g_out.view.view(rows, ldo)
        if ldo > Cn:
            assert bool((bits(full[:, Cn:]) == SENT32).all()), "a store landed in out's row padding"
        res["out"] = full[:, :Cn]
    if planes:
        res["planes"] = g_pl.view.view(2, rows, Cn)
        if planes == 1:
            assert bool((bits(res["planes"][1]) == SENT16).all()), "split_lo = 0 wrote the lo plane"
    if head_out:
        res["head"] = g_head.view
    if dur_out:
        res["dur"] = g_dur.view
    return res


def ln64(v, gamma, beta, eps):
    """float64 LayerNorm of the fp32 rows v: (y64, error scale |gamma| (|x^| + mean|v| / s) + |beta|), s = sqrt(var + eps)."""
    v = v.double()
    mean = v.mean(-1, keepdim=True)
    s = torch.sqrt(((v - mean) ** 2).mean(-1, keepdim=True) + float(F32(eps)))
    xh = (v - mean) / s
    g, b = gamma.double(), beta.double()
    return xh * g + b, g.abs() * (xh.abs() + v.abs().mean(-1, keepdim=True) / s) + b.abs()


def ratio(y, y64, scale):
    return float(((y.double() - y64).abs() / scale).max())


# ---- a. LayerNorm against float64 -------------------------------------------------------------------------------
def families(C, seed):
    """name -> [32, C] fp32 rows."""
    n = 32
    base = rnd((n, C), seed)
    outlier = base.clone()
    outlier[torch.arange(n), torch.arange(n) * 7 % C] = 1e4
    mixed_zero = torch.zeros(n, C, device=DEV)
    mixed_zero[:, ::2] = -0.0
    const = rnd((n, 1), seed + 1, 3.0).expand(n, C).contiguous()
    return {"normal": base, "offset_1e4": base + 1e4, "outlier_1e4": outlier,
            "small_1e-4": base * 1e-4, "small_1e-8": base * 1e-8, "small_1e-19": base * 1e-19,
            "constant": const, "zero": torch.zeros(n, C, device=DEV), "signed_zero": mixed_zero}


@pytest.mark.parametrize("C", [256, 384])
@pytest.mark.parametrize("eps", [1e-5, 1e-12])
def test_layernorm_vs_float64(C, eps):
    gamma, beta = rnd(C, 1), rnd(C, 2)
    err, exact = {}, {}
    for i, (name, x) in enumerate(families(C, 10 + C).items()):
        resid = rnd(x.shape, 100 + i) if name in ("normal", "outlier_1e4") else None
        v = x + resid if resid is not None else x            # fp32, as the kernel adds it
        y = row_norm(x, gamma, beta, eps, resid=resid, ldr=C if resid is not None else None)["out"]
        y64, scale = ln64(v, gamma, beta, eps)
        err[name] = ratio(y, y64, scale)
        measured(f"layernorm_C{C}_eps{eps:g}_{name}", err[name])
        if name in ("zero", "signed_zero") or (name == "constant" and C == 256):
            exact[name] = same_bits(y, beta.expand_as(y))
    assert max(err.values()) <= GATE["layernorm"], err
    assert all(exact.values()), f"rows with no variance must give beta bit for bit: {exact}"


# ---- b. every fusion bit for bit (gamma = 0) --------------------------------------------------------------------
B_, L_, C_ = 4, 37, 256
LENS = [37, 20, 1, 30]
SPK = [2, -1, 4, 0]                  # -1 and n_spk = 4 add nothing
HEAD_C = 129


def fusion_inputs(C=C_, seed=0):
    rows = B_ * L_
    return dict(x=rnd((rows, C), seed), gamma=torch.zeros(C, device=DEV), beta=rnd(C, seed + 1),
                pe=rnd((L_, C), seed + 2), alpha=torch.tensor([0.7381], device=DEV),
                spk_table=rnd((4, C), seed + 3, 0.5), spk=torch.tensor(SPK, device=DEV),
                head_w=torch.nn.functional.one_hot(torch.tensor(HEAD_C), C).float().to(DEV),
                head_b=torch.tensor([0.3141], device=DEV), head_scale=torch.rand(rows, device=DEV) * 1.5 + 0.5,
                lens=torch.tensor(LENS, device=DEV))


FUSIONS = {
    "all": dict(relu=True, pe=True, spk=True, head=True, scale=True, dur=True, lens=True, planes=2),
    "relu": dict(relu=True), "pe": dict(pe=True), "spk": dict(spk=True), "head": dict(head=True),
    "head_scale": dict(head=True, scale=True), "dur": dict(head=True, dur=True), "lens": dict(lens=True),
    "planes": dict(planes=2), "planes_hi_only": dict(planes=1),
}


@pytest.mark.parametrize("case", list(FUSIONS))
def test_fusions_bit_for_bit(case):
    f = FUSIONS[case]
    t = fusion_inputs()
    rows = B_ * L_
    head = f.get("head", False)
    res = row_norm(t["x"], t["gamma"], t["beta"], 1e-5, relu=f.get("relu", False),
                   pe=t["pe"] if f.get("pe") else None, alpha=t["alpha"] if f.get("pe") else None,
                   L=L_ if (f.get("pe") or f.get("lens")) else 0,
                   spk_table=t["spk_table"] if f.get("spk") else None, spk=t["spk"] if f.get("spk") else None,
                   spk_L=L_ if f.get("spk") else 0, head_w=t["head_w"] if head else None, head_b=t["head_b"] if head else None,
                   head_out=head, dur_out=f.get("dur", False), head_scale=t["head_scale"] if f.get("scale") else None,
                   lens=t["lens"] if f.get("lens") else None, planes=f.get("planes", 0))
    npy = lambda k: t[k].cpu().numpy()
    want, want_head, padded = fused_rows(
        npy("beta"), rows, relu=f.get("relu", False), alpha=npy("alpha")[0] if f.get("pe") else None,
        pe=npy("pe") if f.get("pe") else None, L=L_, spk_table=npy("spk_table") if f.get("spk") else None,
        spk=np.array(SPK), spk_L=L_, head_c=HEAD_C if head else None, head_b=npy("head_b")[0] if head else None,
        head_scale=npy("head_scale") if f.get("scale") else None, lens=np.array(LENS) if f.get("lens") else None)
    want = torch.from_numpy(want).to(DEV)
    assert same_bits(res["out"], want), f"{case}: out differs from the fp32 restatement"
    if f.get("planes"):
        sp = split_planes(want, 2)
        assert torch.equal(bits(res["planes"][0]), sp[0]), f"{case}: hi plane"
        if f["planes"] == 2:
            assert torch.equal(bits(res["planes"][1]), sp[1]), f"{case}: lo plane"
    if head:
        assert same_bits(res["head"], torch.from_numpy(want_head).to(DEV)), f"{case}: head"
    if f.get("dur"):
        unscaled = fused_rows(npy("beta"), rows, relu=f.get("relu", False), alpha=npy("alpha")[0] if f.get("pe") else None,
                              pe=npy("pe") if f.get("pe") else None, L=L_, head_c=HEAD_C, head_b=npy("head_b")[0],
                              spk_table=npy("spk_table") if f.get("spk") else None, spk=np.array(SPK), spk_L=L_)[1]
        s = torch.from_numpy(unscaled).to(DEV)
        rule = torch.clamp(torch.round(torch.exp(s) - 1), min=0).long()
        rule[torch.from_numpy(padded).to(DEV)] = 0
        assert torch.equal(res["dur"], rule), f"{case}: dur_out"


# ---- c. the configurations the stages issue, random gamma and beta ----------------------------------------------
def masked_rows(y, lens, L):
    r = torch.arange(y.shape[0], device=DEV)
    return (r % L) >= lens[r // L]


def stage_case(name, C, eps, seed, **kw):
    """Runs one stage configuration and checks it against float64; returns the kernel's results."""
    B, L = 3, 45
    rows = B * L
    x = rnd((rows, C), seed, 2.0, 0.5)
    gamma, beta = rnd(C, seed + 1), rnd(C, seed + 2)
    lens = torch.tensor([45, 17, 1], device=DEV)
    args = dict(kw)
    if args.pop("zlens", False):
        args.update(lens=lens, L=L)
    res = row_norm(x, gamma, beta, eps, **args)
    y64, scale = ln64(x, gamma, beta, eps)
    if args.get("relu"):
        y64 = y64.clamp_min(0)
    if args.get("pe") is not None:
        add = (args["alpha"].double() * args["pe"].double())[torch.arange(rows, device=DEV) % L]
        y64, scale = y64 + add, scale + add.abs()
    if args.get("spk_table") is not None:
        add = args["spk_table"].double()[args["spk"][torch.arange(rows, device=DEV) // args["spk_L"]]]
        y64, scale = y64 + add, scale + add.abs()
    pad = masked_rows(y64, args["lens"], args["L"]) if args.get("lens") is not None else torch.zeros(rows, dtype=torch.bool, device=DEV)
    y64[pad] = 0
    if "out" in res:
        assert bool((bits(res["out"][pad]) == 0).all()), f"{name}: padded rows must be +0"
        measured(f"stage_{name}", ratio(res["out"], y64, scale))
        assert ratio(res["out"], y64, scale) <= GATE["layernorm"]
        if "planes" in res:
            sp = split_planes(res["out"], 2)
            assert torch.equal(bits(res["planes"][0]), sp[0]) and torch.equal(bits(res["planes"][1]), sp[1])
    if "head" in res:
        w, b = args["head_w"].double(), float(args["head_b"])
        h64 = y64 @ w + b
        hscale = (y64 * w).abs().sum(-1) + abs(b)
        got = res["head"].double()
        if args.get("head_scale") is not None:
            h64, hscale = h64 * args["head_scale"].double(), hscale * args["head_scale"].double()
        h64[pad] = 0
        assert bool((bits(res["head"][pad]) == 0).all())
        r = float(((got - h64).abs() / hscale).max())
        measured(f"stage_{name}_head", r)
        assert r <= GATE["head"]
    return res


@pytest.mark.parametrize("C", [256, 384])
def test_stage_fft_block_layernorm(C):
    """FFT-block LayerNorm: out plus hi + lo planes, rows past zlens written as zeros."""
    stage_case(f"fft_block_C{C}", C, 1e-5, 1, planes=2, zlens=True)


def test_stage_last_encoder_layernorm_with_speakers():
    spk_table = rnd((5, 256), 9)
    stage_case("encoder_speaker", 256, 1e-5, 2, planes=2, zlens=True, spk_table=spk_table,
               spk=torch.tensor([3, 0, 4], device=DEV), spk_L=45)


def test_stage_predictor_middle_layernorm():
    """C = 256, eps 1e-12: fp32 out, or hi + lo planes only; the planes-only call writes the same planes."""
    a = stage_case("predictor_mid_out", 256, 1e-12, 3, zlens=True)
    b = stage_case("predictor_mid_planes", 256, 1e-12, 3, zlens=True, out=False, planes=2)
    assert torch.equal(bits(b["planes"]), split_planes(a["out"], 2))


@pytest.mark.parametrize("what", ["dur", "scale"])
def test_stage_predictor_head(what):
    """The last predictor LayerNorm: head only (no out), lens always set; dur_out equals the duration rule applied on the
    device to the kernel's own head_out."""
    head_w, head_b = rnd(256, 20, 0.1), torch.tensor([0.75], device=DEV)
    scale = torch.rand(135, device=DEV) + 0.5 if what == "scale" else None
    res = stage_case(f"predictor_head_{what}", 256, 1e-12, 4, out=False, zlens=True, head_w=head_w, head_b=head_b,
                     head_out=True, dur_out=what == "dur", head_scale=scale)
    if what == "dur":
        rule = torch.clamp(torch.round(torch.exp(res["head"]) - 1), min=0).long()
        assert torch.equal(res["dur"], rule)


def test_stage_decoder_input():
    """relu, then + alpha * pe[t] with L = frames."""
    stage_case("decoder_input", 384, 1e-5, 5, relu=True, pe=rnd((45, 384), 30), alpha=torch.tensor([1.3], device=DEV), L=45,
               planes=2)


@pytest.mark.parametrize("C", [256, 384])
def test_layernorm_entry_equals_row_norm(C):
    """fs2_op_layernorm (the train path's entry): x + resid at 1000 rows, eps 1e-5, against float64 and bit for bit
    equal to fs2_op_row_norm with the same fields."""
    x, r = rnd((1000, C), C, 3.0), rnd((1000, C), C + 1)
    gamma, beta = rnd(C, C + 2), rnd(C, C + 3)
    out = torch.empty(1000, C, device=DEV)
    _lib.check(_lib.load().fs2_op_layernorm(P(x), P(r), P(gamma), P(beta), 1e-5, 1000, C, P(out),
                                             _lib.stream_ptr(out.device)), "fs2_op_layernorm")
    same = row_norm(x, gamma, beta, 1e-5, resid=r, ldr=C)["out"]
    assert same_bits(out, same)
    y64, scale = ln64(x + r, gamma, beta, 1e-5)
    measured(f"layernorm_entry_C{C}", ratio(out, y64, scale))
    assert ratio(out, y64, scale) <= GATE["layernorm"]


# ---- d. the duration rule at its ties ---------------------------------------------------------------------------
def durations_of(xs):
    """dur_out and head_out for head values xs (float32 numpy), driven as gamma = beta = 0, alpha = 1 and pe row t
    carrying xs[t] in channel 0 under a one-hot head_w (head_b = 0); x is one zero row read by every row (ldx = 0)."""
    C = 256
    zero = torch.zeros(C, device=DEV)
    head_w = zero.clone()
    head_w[0] = 1
    one, b0 = torch.ones(1, device=DEV), torch.zeros(1, device=DEV)
    durs, heads = [], []
    for s in range(0, xs.size, 1 << 20):
        chunk = torch.from_numpy(xs[s:s + (1 << 20)]).to(DEV)
        n = chunk.numel()
        pe = torch.zeros(n, C, device=DEV)
        pe[:, 0] = chunk
        res = row_norm(zero.view(1, C), zero, zero, 1e-5, rows=n, ldx=0, out=False, pe=pe, alpha=one, L=n, head_w=head_w,
                       head_b=b0, head_out=True, dur_out=True)
        durs.append(res["dur"].cpu())
        heads.append(res["head"].cpu())
        del pe
    return torch.cat(durs).numpy(), torch.cat(heads).numpy()


def test_duration_rule_at_ties():
    """1. Wherever float64 exp(x) - 1 is more than 2 ulps (expf's error bound) from a tie, dur_out is the float64 truth.
    2. Where exp(x) lies within 0.01 ulp of k + 1.5 and the device's expf returns k + 1.5 itself, dur_out is half to
       even.  expf is not correctly rounded: for some of these x it returns the neighbouring float, and then kernel and
       torch on the same device both round that value (DESIGN.md section 4 lists them).
    3. Everywhere but NaN, dur_out equals the reference's rule evaluated by torch on the same device.  For NaN the
       kernel writes 0 (fmaxf drops the NaN) where torch's .long() on the device gives INT64_MIN."""
    xs = np.concatenate([tie_set(), uniform_set(), special_set(), exact_tie_candidates(TIE_KMAX + 1, 3 * TIE_KMAX)])
    dur, head = durations_of(xs)
    nan = np.isnan(xs)
    fin = ~nan
    assert np.array_equal(head[fin], np.where(xs[fin] == 0, F32(0), xs[fin])), "the head did not carry x"
    with np.errstate(over="ignore", invalid="ignore"):
        e64 = np.exp(xs.astype(np.float64))
    k, d = tie_distance(xs)
    # 1. away from ties (and from the int64 saturation edge): the float64 truth
    far = fin & (((d > 2) & (e64 < 2.0 ** 24)) | (e64 > 2.0 ** 63 * (1 + 2.0 ** -20)) | np.isneginf(xs))
    truth = dur_truth(xs)
    bad = far & (dur != truth)
    measured("duration_far_from_tie_mismatches", float(bad.sum()))
    # 2. exact ties of the device's expf: half to even
    xg = torch.from_numpy(xs).to(DEV)
    dev_exp = torch.exp(xg).cpu().numpy()
    tie = exact_ties(xs)
    dev_tie = tie & (dev_exp == (k + 1.5).astype(F32))
    even = int(np.sum(dev_tie & (k % 2 == 0)))
    tie_bad = dev_tie & (dur != tie_half_even(k).astype(np.int64))
    measured("duration_exact_ties", float(tie.sum()))
    measured("duration_exact_ties_even_k_device_exact", float(even))
    measured("duration_exact_ties_expf_not_exact", float(np.sum(tie & ~dev_tie)))
    # 3. the reference's rule evaluated by torch on the same device (and, reported only, on the CPU)
    gpu_rule = torch.clamp(torch.round(torch.exp(xg) - 1), min=0).long().cpu().numpy()
    cpu_rule = torch.clamp(torch.round(torch.exp(torch.from_numpy(xs)) - 1), min=0).long().numpy()
    dev_bad = fin & (dur != gpu_rule)
    measured("duration_cpu_rule_disagreements", float(np.sum(fin & (dur != cpu_rule))))
    for name, m in (("far", bad), ("tie", tie_bad), ("torch_gpu", dev_bad), ("expf_not_exact", tie & ~dev_tie)):
        if m.any():
            idx = np.flatnonzero(m)[:20]
            print(f"MISMATCH {name}", [(float(xs[i]), hex(int(xs[i:i + 1].view(np.int32)[0])), int(dur[i]), int(truth[i]),
                                       int(gpu_rule[i])) for i in idx])
    assert far.sum() > 2_000_000 and not bad.any()
    assert even >= 20 and not tie_bad.any()
    assert not dev_bad.any()
    assert bool(np.all(dur[nan] == 0))


# ---- e. bucket edges, the variance gather and the one-hot --------------------------------------------------------
@pytest.mark.parametrize("name", list(bin_sets()))
def test_bucketize_and_variance_embed_at_edges(name):
    b = bin_sets()[name]
    n_edges = b.size
    vals = edge_values(b)
    nv = vals.size
    perm = np.random.default_rng(n_edges).permutation(nv)
    want_ids = torch.bucketize(torch.from_numpy(vals), torch.from_numpy(b))
    bins = torch.from_numpy(b).to(DEV)
    lib, st = _lib.load(), _lib.stream_ptr(torch.device(DEV))
    # fs2_bucketize
    ids = torch.full((nv,), SENT64, dtype=torch.int64, device=DEV)
    vals_d = torch.from_numpy(vals).to(DEV)
    _lib.check(lib.fs2_bucketize(P(vals_d), P(bins), n_edges, nv, P(ids), st), "fs2_bucketize")
    assert torch.equal(ids.cpu(), want_ids)
    # fs2_op_variance_embed_add: utterance 0 = the values, utterance 1 = them permuted, padded past nv // 2
    for Cn in (256, 384):
        L, rows = nv, 2 * nv
        lens = torch.tensor([nv, nv // 2], device=DEV)
        e_val = np.concatenate([vals, vals[perm]])
        p_val = np.concatenate([vals[perm], vals])
        e_val_d, p_val_d = torch.from_numpy(e_val).to(DEV), torch.from_numpy(p_val).to(DEV)
        hm = rnd((rows, Cn), 7)
        e_tab, p_tab = rnd((n_edges + 1, Cn), 8), rnd((n_edges + 1, Cn), 9)
        e_bias, p_bias = rnd(Cn, 10), rnd(Cn, 11)
        e_ids_w = torch.bucketize(torch.from_numpy(e_val), torch.from_numpy(b)).numpy()
        p_ids_w = torch.bucketize(torch.from_numpy(p_val), torch.from_numpy(b)).numpy()
        pad = (np.arange(rows) % L) >= np.array([nv, nv // 2])[np.arange(rows) // L]
        want = variance_rows(hm.cpu().numpy(), e_ids_w, p_ids_w, e_tab.cpu().numpy(), e_bias.cpu().numpy(), p_tab.cpu().numpy(),
                             p_bias.cpu().numpy())
        want[pad] = 0
        want = torch.from_numpy(want).to(DEV)
        e_ids_w[pad], p_ids_w[pad] = -1, -1
        for mode in ("out+lo", "hi_only"):
            g_out = Guarded(rows * Cn, torch.float32)
            g_pl = Guarded(2 * rows * Cn, torch.float16)
            g_e, g_p = Guarded64(rows), Guarded64(rows)
            _lib.check(lib.fs2_op_variance_embed_add(
                P(hm), P(e_val_d), P(p_val_d), P(bins), P(bins), n_edges,
                P(e_tab), P(e_bias), P(p_tab), P(p_bias), rows, Cn, P(g_out.view) if mode == "out+lo" else None, P(g_pl.view),
                int(mode == "out+lo"), P(g_e.view), P(g_p.view), P(lens), L, st), "fs2_op_variance_embed_add")
            torch.cuda.synchronize()
            assert g_out.intact() and g_pl.intact() and g_e.intact() and g_p.intact()
            assert np.array_equal(g_e.view.cpu().numpy(), e_ids_w) and np.array_equal(g_p.view.cpu().numpy(), p_ids_w)
            pl = g_pl.view.view(2, rows, Cn)
            sp = split_planes(want, 2)
            assert torch.equal(bits(pl[0]), sp[0])
            if mode == "out+lo":
                assert same_bits(g_out.view.view(rows, Cn), want), "out != (h + (pw + pb)) + (ew + eb)"
                assert torch.equal(bits(pl[1]), sp[1])
            else:
                assert bool((bits(g_out.view) == SENT32).all()) and bool((bits(pl[1]) == SENT16).all())
    # fs2_one_hot of -1 (padding) and of n_edges
    n_bins = (n_edges + 1 + 3) // 4 * 4
    oh_ids = torch.tensor([-1, n_edges, 0, n_edges // 2, -1], device=DEV)
    g = Guarded(oh_ids.numel() * n_bins, torch.float32)
    _lib.check(lib.fs2_one_hot(P(oh_ids), oh_ids.numel(), n_bins, P(g.view), st), "fs2_one_hot")
    torch.cuda.synchronize()
    assert g.intact()
    oh = g.view.view(-1, n_bins)
    want_oh = torch.nn.functional.one_hot(oh_ids.clamp_min(0), n_bins).float()
    want_oh[oh_ids < 0] = 0
    assert same_bits(oh, want_oh)


# ---- f. the encoder input embedding, inference form -------------------------------------------------------------
@pytest.mark.parametrize("C", [256, 384])
def test_embed_posenc_inference_form(C):
    B, T, n_sym = 3, 45, 20
    xs = torch.randint(0, n_sym, (B, T), generator=torch.Generator().manual_seed(C))
    xs[0, :4] = torch.tensor([-1, n_sym, n_sym + 5, -7])
    xs = xs.to(DEV)
    table, pe, alpha = rnd((n_sym, C), 1), rnd((T, C), 2), torch.tensor([0.6173], device=DEV)
    lens = torch.tensor([45, 17, 1], device=DEV)
    g_out, g_pl = Guarded(B * T * C, torch.float32), Guarded(2 * B * T * C, torch.float16)
    _lib.check(_lib.load().fs2_embed_posenc(P(xs), P(table), n_sym, P(pe), P(alpha), B, T, C, P(g_out.view), P(g_pl.view),
                                            P(lens), _lib.stream_ptr(torch.device(DEV))), "fs2_embed_posenc")
    torch.cuda.synchronize()
    assert g_out.intact() and g_pl.intact()
    ids = torch.where((xs < 0) | (xs >= n_sym), 0, xs).cpu().numpy().ravel()
    t = np.arange(B * T) % T
    want = (table.cpu().numpy()[ids] + (F32(alpha.item()) * pe.cpu().numpy()[t]).astype(F32)).astype(F32)
    want[t >= lens.cpu().numpy()[np.arange(B * T) // T]] = 0
    want = torch.from_numpy(want).to(DEV)
    assert same_bits(g_out.view.view(B * T, C), want)
    assert torch.equal(bits(g_pl.view.view(2, B * T, C)), split_planes(want, 2))


# ---- g. padding, per-utterance independence and geometry ---------------------------------------------------------
def full_fusion_call(x, resid, spk, lens, t, L, C, **kw):
    return row_norm(x, t["gamma"], t["beta"], 1e-5, resid=resid, ldr=C, relu=True, pe=t["pe"], alpha=t["alpha"], L=L,
                    spk_table=t["spk_table"], spk=spk, spk_L=L, head_w=t["head_w"], head_b=t["head_b"], head_out=True,
                    dur_out=True, lens=lens, planes=2, **kw)


def test_padding_nan_and_per_utterance_independence():
    """NaN in x and resid past lens changes no valid bit; each utterance alone and the reversed batch give the same bits
    (this pins pe[row % L] and spk[row / spk_L])."""
    C = 384
    t = fusion_inputs(C, 40)
    t["gamma"] = rnd(C, 41)
    t["head_w"] = rnd(C, 42, 0.1)
    rows = B_ * L_
    x, resid = t["x"], rnd((rows, C), 43)
    spk = torch.tensor([2, 1, 3, 0], device=DEV)
    lens = t["lens"]
    pad = masked_rows(x, lens, L_)
    base = full_fusion_call(x, resid, spk, lens, t, L_, C)
    xn, rn = x.clone(), resid.clone()
    xn[pad], rn[pad] = float("nan"), float("nan")
    nan = full_fusion_call(xn, rn, spk, lens, t, L_, C)
    for k in base:
        assert same_bits(base[k], nan[k]), k
    assert bool((bits(base["out"][pad]) == 0).all()) and bool((base["dur"][pad] == 0).all())
    for b in range(B_):
        sl = slice(b * L_, (b + 1) * L_)
        one = full_fusion_call(xn[sl].contiguous(), rn[sl].contiguous(), spk[b:b + 1].contiguous(), lens[b:b + 1].contiguous(),
                               t, L_, C)
        for k in ("out", "head", "dur"):
            assert same_bits(one[k], nan[k][sl]), (b, k)
        assert torch.equal(bits(one["planes"]), bits(nan["planes"][:, sl])), b
    rev = lambda v: v.view(B_, L_, *v.shape[1:]).flip(0).reshape(v.shape)
    r = full_fusion_call(rev(xn).contiguous(), rev(rn).contiguous(), spk.flip(0).contiguous(), lens.flip(0).contiguous(), t, L_, C)
    for k in ("out", "head", "dur"):
        assert same_bits(rev(r[k]), nan[k]), k


def test_variance_embed_nan_padding():
    C, B, L = 256, 3, 40
    rows = B * L
    bins = torch.from_numpy(bin_sets()["pitch"]).to(DEV)
    lens = torch.tensor([40, 9, 1], device=DEV)
    hm, e_val, p_val = rnd((rows, C), 1), rnd(rows, 2, 100, 200), rnd(rows, 3, 100, 200)
    tabs = [rnd((256, C), 4), rnd(C, 5), rnd((256, C), 6), rnd(C, 7)]
    pad = masked_rows(hm, lens, L)

    def call(h, e, p):
        out = torch.empty(rows, C, device=DEV)
        ei, pi = torch.empty(rows, dtype=torch.int64, device=DEV), torch.empty(rows, dtype=torch.int64, device=DEV)
        _lib.check(_lib.load().fs2_op_variance_embed_add(P(h), P(e), P(p), P(bins), P(bins), 255, *[P(v) for v in tabs], rows, C,
                                                         P(out), None, 0, P(ei), P(pi), P(lens), L,
                                                         _lib.stream_ptr(torch.device(DEV))), "fs2_op_variance_embed_add")
        torch.cuda.synchronize()
        return out, ei, pi
    a = call(hm, e_val, p_val)
    hn, en, pn = hm.clone(), e_val.clone(), p_val.clone()
    hn[pad], en[pad], pn[pad] = float("nan"), float("nan"), float("nan")
    b = call(hn, en, pn)
    assert same_bits(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    assert bool((bits(a[0][pad]) == 0).all()) and bool((a[1][pad] == -1).all())


@pytest.mark.parametrize("rows", [1, 7, 8, 9, 8 * 132 + 1, 51203])
@pytest.mark.parametrize("C", [256, 384])
def test_row_tails_and_strides(rows, C):
    """Tails of the 8-rows-per-CTA grid, with row strides ldx, ldr and ldo different from C."""
    ldx, ldr, ldo = C + 4, C + 8, C + 12
    x = rnd((rows, ldx), rows + C, 2.0)
    resid = rnd((rows, ldr), rows + C + 1)
    gamma, beta = rnd(C, 3), rnd(C, 4)
    y = row_norm(x, gamma, beta, 1e-5, resid=resid, ldr=ldr, ldo=ldo)["out"]
    y64, scale = ln64(x[:, :C] + resid[:, :C], gamma, beta, 1e-5)
    r = ratio(y, y64, scale)
    measured(f"tails_C{C}", r)
    assert r <= GATE["layernorm"]


def test_more_than_2_31_elements():
    """C = 256 rows past 2^31 elements (row * C overflows int32): sampled rows against float64."""
    C = 256
    rows = (1 << 31) // C + 37
    need = 2 * rows * C * 4 + (1 << 30)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        print(f"SKIPPED more_than_2_31_elements: {free / 1e9:.1f} GB free, {need / 1e9:.1f} GB needed")
        pytest.skip("not enough free device memory")
    x = torch.empty(rows, C, device=DEV)
    x.normal_(generator=torch.Generator(device=DEV).manual_seed(5))
    gamma, beta = rnd(C, 6), rnd(C, 7)
    out = torch.empty(rows, C, device=DEV)
    d = _lib.RowNormDesc(x=P(x), ldx=C, gamma=P(gamma), beta=P(beta), eps=1e-5, rows=rows, C=C, out=P(out), ldo=C)
    _lib.check(_lib.load().fs2_op_row_norm(ctypes.byref(d), _lib.stream_ptr(torch.device(DEV))), "fs2_op_row_norm")
    torch.cuda.synchronize()
    sample = torch.cat([torch.arange(64, device=DEV), torch.arange(rows - 4096, rows, device=DEV),
                        torch.randint(0, rows, (4096,), device=DEV, generator=torch.Generator(device=DEV).manual_seed(8))])
    y64, scale = ln64(x[sample], gamma, beta, 1e-5)
    r = ratio(out[sample], y64, scale)
    measured("rows_past_2_31", r)
    assert r <= GATE["layernorm"]
