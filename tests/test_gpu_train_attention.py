"""The fused tf32 train attention on the GPU (DESIGN.md §13, csrc/attention_train_tc.cu, train_attention="flash").

* the kernels against float64, on their own tf32-rounded operands (tight) and on the exact operands, at dk 128 / 192,
  L from 1 to 800 with lens 0, 1, L - 1, L and ragged in one batch, p = 0 and 0.2 (explicit mask);
* the (seed, offset) path against the explicit mask fs2_dropout_mask draws, bit for bit;
* padding: NaN past len and in the workspace, zeros past len, guard bands, determinism; per-utterance independence;
* memory: nothing O(L^2) at L = 8192;
* the model step against the reference's autograd (golden, masks injected), flash against materialized with Philox
  masks, the optimizer recipe, and eval unaffected.
Error metric: max |err| / sum |terms| per output element.  Gates are about 3x the worst observed; observed values are in
DESIGN.md §13.  Needs an H100: run with `-m gpu`."""
import json
import math

import pytest
import torch

from fastspeech2_b200 import FeedForwardTransformer, _lib
from fastspeech2_b200 import train as T
from fastspeech2_b200.hparams import load_hp
from fastspeech2_b200.synthetic import make_batch

pytestmark = pytest.mark.gpu
KEYS = ("xs", "ilens", "ys", "olens", "ds", "es", "ps")
GUARD = 64
SENTINEL = 12345.5


def tf32_rna(t):
    """cvt.rna.tf32.f32: round the fp32 mantissa to 10 bits, to nearest, ties away from zero."""
    b = t.contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


def _st():
    return torch.cuda.current_stream().cuda_stream


def run(q, k, v, dout, lens, heads, p, dmask=None, seed=0, offset=0, ws=None, outs=None):
    """Forward and backward through the C ABI; returns (out, lse, dq, dk, dv)."""
    lib = _lib.load()
    B, L, C = q.shape
    nbytes = T.attn_train_ws_bytes(B, L, C, heads)
    if ws is None:
        ws = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    if outs is None:
        outs = [torch.empty(B, L, C, device="cuda"), torch.empty(B * heads, L, device="cuda")] + [torch.empty(B, L, C, device="cuda") for _ in range(3)]
    out, lse, dq, dk, dv = outs
    mp = None if dmask is None else dmask.data_ptr()
    _lib.check(lib.fs2_attn_train_forward(q.data_ptr(), k.data_ptr(), v.data_ptr(), lens.data_ptr(), B, L, C, heads, float(p), mp, seed, offset,
                                          out.data_ptr(), lse.data_ptr(), ws.data_ptr(), nbytes, _st()), "fs2_attn_train_forward")
    _lib.check(lib.fs2_attn_train_backward(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(), dout.data_ptr(), lens.data_ptr(),
                                           B, L, C, heads, float(p), mp, seed, offset, dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), ws.data_ptr(),
                                           nbytes, _st()), "fs2_attn_train_backward")
    torch.cuda.synchronize()
    return out, lse, dq, dk, dv


def reference(q, k, v, dout, lens, heads, p, dmask):
    """float64: (O, lse, dQ, dK, dV) and the sums of |terms| of each output element."""
    B, L, C = q.shape
    dk = C // heads
    sh = lambda t: t.double().reshape(B, L, heads, dk).permute(0, 2, 1, 3)     # [B, h, L, dk]
    q, k, v, do = sh(q), sh(k), sh(v), sh(dout)
    scale = 1.0 / math.sqrt(dk)
    idx = torch.arange(L, device=q.device)
    valid = (idx[None, :] < lens[:, None]).view(B, 1, L, 1) & (idx[None, :] < lens[:, None]).view(B, 1, 1, L)
    s = torch.einsum("bhid,bhjd->bhij", q, k) * scale
    s = s.masked_fill(~valid, -math.inf)
    mx = s.amax(-1, keepdim=True).clamp_min(-1e300)
    e = torch.exp(s - mx)
    den = e.sum(-1, keepdim=True)
    P = torch.where(valid, e / den.clamp_min(1e-300), torch.zeros_like(e))
    lse = torch.where(valid.any(-1), (mx + torch.log(den.clamp_min(1e-300))).squeeze(-1), torch.zeros_like(mx.squeeze(-1)))
    M = torch.ones_like(P) if dmask is None else dmask.double() / (1.0 - p)
    Pd = P * M
    O = torch.einsum("bhij,bhjd->bhid", Pd, v)
    Oa = torch.einsum("bhij,bhjd->bhid", Pd.abs(), v.abs())
    dV = torch.einsum("bhij,bhid->bhjd", Pd, do)
    dVa = torch.einsum("bhij,bhid->bhjd", Pd.abs(), do.abs())
    dP = torch.einsum("bhid,bhjd->bhij", do, v) * M
    D = (dP * P).sum(-1, keepdim=True)
    dS = P * (dP - D)
    dSa = P * (dP.abs() + (P * dP.abs()).sum(-1, keepdim=True))          # the terms of dS, D's included
    dQ = torch.einsum("bhij,bhjd->bhid", dS, k) * scale
    dQa = torch.einsum("bhij,bhjd->bhid", dSa, k.abs()) * scale
    dK = torch.einsum("bhij,bhid->bhjd", dS, q) * scale
    dKa = torch.einsum("bhij,bhid->bhjd", dSa, q.abs()) * scale
    back = lambda t: t.permute(0, 2, 1, 3).reshape(B, L, C)
    return [back(O), lse.reshape(B * heads, L), back(dQ), back(dK), back(dV)], [back(Oa), None, back(dQa), back(dKa), back(dVa)]


def metrics(got, want, terms):
    errs = []
    for g, w, a in zip(got, want, terms):
        d = (g.double() - w).abs()
        if a is None:
            errs.append(float((d / (1.0 + w.abs())).max()))
        else:
            errs.append(float((d / (a + 1e-30)).max()))
    return errs


def make_inputs(B, L, dk, heads, seed, lens):
    g = torch.Generator().manual_seed(seed)
    C = dk * heads
    q, k, v, do = (torch.randn(B, L, C, generator=g) for _ in range(4))
    q = q * 1.5
    return [t.cuda() for t in (q, k, v, do)] + [torch.tensor(lens, dtype=torch.int64, device="cuda")]


LS = [1, 5, 63, 64, 65, 127, 128, 129, 200, 800]
# Gates per output (O, lse, dQ, dK, dV), at most 3x the worst observed on the first H100 run (DESIGN.md §13), against
# float64 on the rna-rounded operands and on the exact ones.  dQ / dK come out larger: dS = P (dP - D) is small where dP
# and D nearly cancel, while its error follows the tf32 rounding of the dO.V^T operands and of dS itself.
OUTPUTS = ("O", "lse", "dQ", "dK", "dV")
TIGHT_GATES = (1.3e-3, 1.6e-6, 1e-2, 1e-2, 1.25e-3)
EXACT_GATES = (4.5e-3, 2.4e-3, 7.2e-2, 1e-2, 6e-3)


@pytest.mark.parametrize("p", [0.0, 0.2])
@pytest.mark.parametrize("L", LS)
@pytest.mark.parametrize("dk", [128, 192])
def test_kernels_against_float64(dk, L, p):
    heads = 2
    lens = [0, 1, max(L - 1, 0), L, L // 2 + 1 if L > 1 else 1]
    B = len(lens)
    q, k, v, do, lt = make_inputs(B, L, dk, heads, 7 * L + dk, lens)
    dmask = None
    if p > 0:
        dmask = (torch.rand(B, heads, L, L, generator=torch.Generator().manual_seed(L)) >= p).to(torch.uint8).cuda()
    got = run(q, k, v, do, lt, heads, p, dmask=dmask)
    want_r, terms = reference(tf32_rna(q), tf32_rna(k), tf32_rna(v), tf32_rna(do), lt, heads, p, dmask)
    want, _ = reference(q, k, v, do, lt, heads, p, dmask)
    tight, exact = metrics(got, want_r, terms), metrics(got, want, terms)
    print(f"dk {dk} L {L} p {p}: O/lse/dQ/dK/dV vs rounded {['%.1e' % e for e in tight]}, vs exact {['%.1e' % e for e in exact]}")
    assert all(torch.isfinite(t).all() for t in got)
    for name, e, gate in zip(OUTPUTS, tight, TIGHT_GATES):
        assert e <= gate, (name, "rounded operands", e, gate)
    for name, e, gate in zip(OUTPUTS, exact, EXACT_GATES):
        assert e <= gate, (name, "exact operands", e, gate)


@pytest.mark.parametrize("case", [(1, 33, 128, 0), (3, 70, 192, (1 << 32) - 1000), (2, 129, 128, 12345)], ids=str)
def test_philox_regeneration_matches_the_explicit_mask(case):
    """(seed, offset) gives the bits of the explicit mask fs2_dropout_mask draws: an element count that is not a multiple
    of 4 (1 x 1 x 33 x 33) and counters that carry into the high word."""
    B, L, dk, offset = case
    heads = 384 // dk if dk == 192 else 1
    lens = [L] + [L - 7 * i for i in range(1, B)]
    q, k, v, do, lt = make_inputs(B, L, dk, heads, L, lens)
    n = B * heads * L * L
    p, seed = 0.2, 0x123456789
    mask = torch.empty(B, heads, L, L, dtype=torch.uint8, device="cuda")
    _lib.check(_lib.load().fs2_dropout_mask(mask.data_ptr(), n, p, seed, offset, _st()), "fs2_dropout_mask")
    a = run(q, k, v, do, lt, heads, p, dmask=mask)
    b = run(q, k, v, do, lt, heads, p, seed=seed, offset=offset)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    c = run(q, k, v, do, lt, heads, p, seed=seed, offset=offset + 1)
    assert not torch.equal(a[0], c[0]), "the offset reaches the mask"


@pytest.mark.parametrize("dk", [128, 192])
def test_padding_nan_guard_bands_and_determinism(dk):
    heads, L = 2, 150
    lens = [150, 97, 0, 64]
    B, C = len(lens), dk * heads
    q, k, v, do, lt = make_inputs(B, L, dk, heads, 11, lens)
    p, seed, offset = 0.2, 99, 4321
    ref = run(q, k, v, do, lt, heads, p, seed=seed, offset=offset)
    qn, kn, vn, dn = (t.clone() for t in (q, k, v, do))
    for b, n in enumerate(lens):
        for t in (qn, kn, vn, dn):
            t[b, n:] = float("nan")
    nbytes = T.attn_train_ws_bytes(B, L, C, heads)
    ws = torch.full((nbytes // 4,), float("nan"), device="cuda").view(torch.uint8)
    sizes = [B * L * C, B * heads * L, B * L * C, B * L * C, B * L * C]
    bufs = [torch.full((n + 2 * GUARD,), SENTINEL, device="cuda") for n in sizes]
    outs = [bf[GUARD:GUARD + n].view(*(r.shape)) for bf, n, r in zip(bufs, sizes, ref)]
    got = run(qn, kn, vn, dn, lt, heads, p, seed=seed, offset=offset, ws=ws, outs=outs)
    for bf, n in zip(bufs, sizes):
        assert (bf[:GUARD] == SENTINEL).all() and (bf[GUARD + n:] == SENTINEL).all()
    for x, y in zip(ref, got):
        assert torch.isfinite(x).all()
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    out, lse, dq, dkk, dv = ref
    for b, n in enumerate(lens):
        for t in (out, dq, dkk, dv):
            assert (t[b, n:].view(torch.int32) == 0).all()
        assert (lse.view(B, heads, L)[b, :, n:].view(torch.int32) == 0).all()
    again = run(q, k, v, do, lt, heads, p, seed=seed, offset=offset)
    for x, y in zip(ref, again):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))


@pytest.mark.parametrize("dk", [128, 192])
def test_per_utterance_independence(dk):
    heads, n = 2, 137
    lens = [n, 300, 211]
    B, L = len(lens), max(lens)
    q, k, v, do, lt = make_inputs(B, L, dk, heads, 5, lens)
    batch = run(q, k, v, do, lt, heads, 0.0)
    alone = run(*(t[:1, :n].contiguous() for t in (q, k, v, do)), lt[:1].clone(), heads, 0.0)
    for x, y in zip(batch[:1] + batch[2:], alone[:1] + alone[2:]):
        assert torch.equal(x[0, :n].view(torch.int32), y[0].view(torch.int32))
    assert torch.equal(batch[1].view(B, heads, L)[0, :, :n], alone[1].view(1, heads, n)[0])


def test_memory_is_linear_in_L():
    B, heads, L, dk = 1, 2, 8192, 192
    C = heads * dk
    q, k, v, do, lt = make_inputs(B, L, dk, heads, 3, [L])
    for t in (q, k, v):
        t.requires_grad_()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = T.FlashAttentionFn.apply(q, k, v, lt, heads, 0.2, None, 7, 0)
    out.backward(do)
    torch.cuda.synchronize()
    rise = torch.cuda.max_memory_allocated() - base
    returned = 4 * out.numel() * 4                       # out, dq, dk, dv
    ws = T.attn_train_ws_bytes(B, L, C, heads)
    lse = B * heads * L * 4
    scores = B * heads * L * L * 4
    print(f"peak rise {rise / 1e6:.1f} MB, returned {returned / 1e6:.1f} MB, workspace {ws / 1e6:.1f} MB, lse {lse / 1e6:.2f} MB, "
          f"one [B, h, L, L] fp32 tensor {scores / 1e6:.0f} MB")
    assert rise - returned <= ws + lse
    assert rise - returned < scores / 4


# ---- the model -----------------------------------------------------------------------------------------------------------------
class _Recorded(T.MaskSource):
    """The reference's masks in call order, permuted to this path's layout where it drops a [B, C, time] tensor; the flash
    attention sites take theirs as explicit masks."""

    def __init__(self, masks):
        super().__init__(seed=0, injected=None)
        self.recorded = list(masks)

    def next(self, shape, p, device):
        self.calls += 1
        m = self.recorded.pop(0)
        if tuple(m.shape) != tuple(shape):
            assert m.dim() == 3 and tuple(m.permute(0, 2, 1).shape) == tuple(shape), (self.calls, tuple(m.shape), tuple(shape))
            m = m.permute(0, 2, 1)
        return m.to(torch.uint8).contiguous().to(device)

    def attention(self, shape, p, device):
        return self.next(shape, p, device), 0, 0


def _model(weights, train_attention, precision="fp32"):
    m = FeedForwardTransformer(68, 80, load_hp(), precision=precision, train_precision="tf32", train_attention=train_attention)
    m.load_state_dict(weights, strict=True)
    return m.cuda()


def _golden_step(weights, golden, ragged):
    g = golden("train_step_ragged" if ragged else "train_step")
    bt = make_batch(3, 23, 181, seed=17, ilens=[23, 17, 9], olens=[181, 140, 66]) if ragged else make_batch(2, 20, 150, seed=16)
    gen = torch.Generator().manual_seed(5)
    recorded = [torch.rand(shape, generator=gen) >= p for shape, p in zip(json.loads(str(g["mask_shapes"])), g["mask_rates"].tolist())]
    m = _model(weights, "flash").train()
    m.dropout_masks = _Recorded(recorded)
    calls = []
    apply = T.FlashAttentionFn.apply

    def counting(*a):
        calls.append(a[0].shape)
        return apply(*a)
    T.FlashAttentionFn.apply = counting
    try:
        loss, rep = m(*[bt[k].cuda() for k in KEYS])
    finally:
        del T.FlashAttentionFn.apply
    loss.backward()
    torch.cuda.synchronize()
    assert not m.dropout_masks.recorded
    assert len(calls) == 8, "every encoder and decoder layer ran the fused attention"
    return g, m, loss, rep


# Gates from the first H100 run (DESIGN.md §13), about 3x the observed worst of the two batches
LOSS_GATE, REPORT_GATE, GRAD_GATE, ALPHA_GATE, KBIAS_GATE, BUF_GATE = 1.5e-6, 7.5e-4, 0.26, 0.25, 1.3e-3, 1.35e-3


@pytest.mark.parametrize("ragged", [False, True])
def test_flash_train_step_matches_reference_autograd(weights, golden, ragged):
    g, m, loss, rep = _golden_step(weights, golden, ragged)
    loss_ref = float(g["loss"])
    lerr = abs(float(loss) - loss_ref) / abs(loss_ref)
    rerr = max(abs(list(a.values())[0] - vb) / max(1.0, abs(vb)) for a, vb in zip(rep, g["report_values"].tolist()))
    no_grad = set(json.loads(str(g["no_grad"])))
    errs, kbias = {}, 0.0
    for name, p in m.named_parameters():
        if name in no_grad:
            assert p.grad is None, name
            continue
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
        flat = p.grad.detach().reshape(-1).cpu()
        scale = float(g["gmax/" + name])
        idx = torch.from_numpy(g["gidx/" + name].astype("int64"))
        err = float((flat[idx] - torch.from_numpy(g["gval/" + name])).abs().max())
        err = max(err, abs(float(flat.abs().max()) - scale))
        if name.endswith("self_attn.linear_k.bias"):
            kbias = max(kbias, err / float(g["gmax/" + name.replace(".bias", ".weight")]))
            continue
        errs[name] = err / (scale + 1e-12)
    alpha = max(errs.pop(n) for n in list(errs) if n.endswith(".alpha"))
    worst = max(errs.items(), key=lambda kv: kv[1])
    bufs = dict(m.named_buffers())
    berr = 0.0
    for key in g:
        if key.startswith("buf/"):
            ref = torch.from_numpy(g[key]).double()
            berr = max(berr, float((bufs[key[4:]].cpu().double() - ref).abs().max() / (ref.abs().max() + 1e-12)))
    print(f"loss rel {lerr:.2e}, report rel {rerr:.2e}, worst gradient {worst[0]} {worst[1]:.2e}, alpha {alpha:.2e}, key bias {kbias:.2e}, "
          f"buffers {berr:.2e}")
    print("largest gradient errors:", sorted(errs.items(), key=lambda kv: -kv[1])[:6])
    assert lerr <= LOSS_GATE and rerr <= REPORT_GATE
    assert worst[1] <= GRAD_GATE, worst
    assert alpha <= ALPHA_GATE and kbias <= KBIAS_GATE and berr <= BUF_GATE


# flash against materialized with Philox masks; gates about 3x the first H100 run's differences (DESIGN.md §13)
FM_LOSS_GATE, FM_NORM_GATE = 4e-7, 1.3e-3


@pytest.mark.parametrize("ragged", [False, True])
def test_flash_against_materialized_with_philox_masks(weights, ragged):
    bt = make_batch(3, 23, 181, seed=17, ilens=[23, 17, 9], olens=[181, 140, 66]) if ragged else make_batch(2, 20, 150, seed=16)
    res = []
    for mode in ("materialized", "flash"):
        m = _model(weights, mode).train()
        m.dropout_masks = T.MaskSource(seed=2024)
        loss, _ = m(*[bt[k].cuda() for k in KEYS])
        loss.backward()
        norm = torch.sqrt(sum((p.grad.double() ** 2).sum() for p in m.parameters() if p.grad is not None))
        res.append((float(loss), float(norm), m.dropout_masks.offset, m.dropout_masks.calls))
    (l0, n0, o0, c0), (l1, n1, o1, c1) = res
    print(f"loss {l0:.7g} / {l1:.7g} rel {abs(l1 - l0) / abs(l0):.2e}; grad norm {n0:.7g} / {n1:.7g} rel {abs(n1 - n0) / n0:.2e}")
    assert (o0, c0) == (o1, c1), "both paths advance the Philox offset alike"
    assert abs(l1 - l0) / abs(l0) <= FM_LOSS_GATE
    assert abs(n1 - n0) / n0 <= FM_NORM_GATE


def test_flash_optimizer_step_through_the_reference_training_recipe(weights):
    m = _model(weights, "flash")
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    args = [make_batch(2, 20, 150, seed=21)[k].cuda() for k in KEYS]
    m.eval()
    with torch.no_grad():
        l0, _ = m(*args)
    m.train()
    for _ in range(3):
        loss, _ = m(*args)
        loss.backward()
        assert math.isfinite(float(torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0)))
        opt.step(); opt.zero_grad()
    m.eval()
    with torch.no_grad():
        l1, _ = m(*args)
    assert float(l1) < float(l0), (float(l0), float(l1))


@pytest.mark.parametrize("precision", ["3xf16", "tf32", "fp32"])
def test_eval_is_unaffected_by_train_attention(weights, precision):
    bt = make_batch(3, 23, 181, seed=17, ilens=[23, 17, 9], olens=[181, 140, 66])
    outs = []
    for mode in ("materialized", "flash"):
        m = _model(weights, mode, precision).eval()
        with torch.no_grad():
            outs.append(m._forward(*[bt[k].cuda() for k in ("xs", "ilens", "olens", "ds", "es", "ps")], is_inference=False))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
