"""The tf32 train mode on the GPU (DESIGN.md §10).

* the tensor-core weight-gradient kernel (fs2_conv_wgrad_tc) on every (N, K, taps) the train step issues and at the edges
  of its work decomposition (tests/_wgrad_plan.py): against float64 on its own tf32-rounded operands (a tight gate: fp32
  accumulation is the only error left) and against exact float64 (a TF32 gate); guard bands, +=, NaN in the unread
  columns of its workspace, determinism;
* ConvFn in tf32 against float64 autograd;
* the model's train step in tf32 against the reference's autograd (tests/golden/train_step*.npz, masks injected as in
  tests/test_gpu_train.py), the optimizer recipe, and an eval path unaffected by the train mode.
Gates are relative to sum_t |dy| |x| (kernel) or to the largest reference value (ConvFn, model); observed values are in
DESIGN.md §10.  Needs an H100: run with `-m gpu`."""
import json
import math

import pytest
import torch

from _wgrad_plan import KERNEL_CASES, TRAIN_SHAPES, ws_bytes
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


def ref_wgrad(dy, x, taps):
    """float64 dW [N, K, taps] and sum |dy| |x| of the same terms."""
    B, L, N = dy.shape
    pad = (taps - 1) // 2
    dy, x = dy.double(), x.double()
    xp = torch.nn.functional.pad(x, (0, 0, pad, pad))
    w = torch.empty(N, x.shape[2], taps, dtype=torch.float64, device=dy.device)
    a = torch.empty_like(w)
    for j in range(taps):
        xs = xp[:, j:j + L]
        w[:, :, j] = torch.einsum("btn,btk->nk", dy, xs)
        a[:, :, j] = torch.einsum("btn,btk->nk", dy.abs(), xs.abs())
    return w, a


def run_wgrad(dy, x, taps, dw=None, ws=None, dbias=None):
    B, L, N = dy.shape
    K = x.shape[2]
    nbytes = ws_bytes(B, L, N, K, taps)
    assert nbytes == T.wgrad_tc_ws_bytes(B, L, N, K, taps)
    if ws is None:
        ws = torch.zeros(max(nbytes, 1), dtype=torch.uint8, device="cuda")
    if dw is None:
        dw = torch.zeros(N, K, taps, device="cuda")
    _lib.check(_lib.load().fs2_conv_wgrad_tc(dy.data_ptr(), x.data_ptr(), B, L, N, K, taps, dw.data_ptr(),
                                             None if dbias is None else dbias.data_ptr(), ws.data_ptr(), nbytes,
                                             torch.cuda.current_stream().cuda_stream), "fs2_conv_wgrad_tc")
    return dw


def inputs(case, seed):
    B, L, N, K, taps = case
    g = torch.Generator().manual_seed(seed)
    dy = torch.randn(B, L, N, generator=g)
    x = torch.randn(B, L, K, generator=g) * 0.5 + 0.1
    return dy.cuda(), x.cuda()


# ---- the kernel -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", KERNEL_CASES, ids=lambda c: "B%d_L%d_N%d_K%d_t%d" % c)
def test_wgrad_kernel_against_float64(case):
    B, L, N, K, taps = case
    dy, x = inputs(case, sum(case))
    got = run_wgrad(dy, x, taps).double()
    want_r, scale = ref_wgrad(tf32_rna(dy), tf32_rna(x), taps)
    want, _ = ref_wgrad(dy, x, taps)
    tight = float(((got - want_r).abs() / (scale + 1e-30)).max())
    loose = float(((got - want).abs() / (scale + 1e-30)).max())
    print(f"{case}: vs rounded operands {tight:.2e}, vs exact {loose:.2e}")
    assert tight <= 2e-6, tight
    assert loose <= 1e-3, loose


def test_wgrad_kernel_guard_bands_and_accumulation():
    case = (3, 45, 80, 256, 5)
    B, L, N, K, taps = case
    dy, x = inputs(case, 1)
    n = N * K * taps
    buf = torch.full((n + 2 * GUARD,), SENTINEL, device="cuda")
    dw0 = torch.randn(n, generator=torch.Generator().manual_seed(2)).cuda()
    buf[GUARD:GUARD + n] = dw0
    db = torch.full((N + 2 * GUARD,), SENTINEL, device="cuda")
    db[GUARD:GUARD + N] = 0.5
    run_wgrad(dy, x, taps, dw=buf[GUARD:], dbias=db[GUARD:])
    torch.cuda.synchronize()
    assert (buf[:GUARD] == SENTINEL).all() and (buf[GUARD + n:] == SENTINEL).all()
    assert (db[:GUARD] == SENTINEL).all() and (db[GUARD + N:] == SENTINEL).all()
    fresh = run_wgrad(dy, x, taps).reshape(-1)
    assert torch.equal(buf[GUARD:GUARD + n], dw0 + fresh), "dw += the same partial sums"
    want_db = 0.5 + dy.double().sum((0, 1))
    assert float((db[GUARD:GUARD + N].double() - want_db).abs().max()) <= 1e-4 * float(want_db.abs().max())


@pytest.mark.parametrize("case", [(3, 45, 80, 256, 5), (5, 1, 256, 80, 5), (16, 201, 1024, 384, 9)], ids=str)
def test_wgrad_kernel_never_reads_past_L_and_is_deterministic(case):
    """NaN in every workspace byte (including the transposed buffers' columns [L, Lp)) changes no bit; two calls agree."""
    B, L, N, K, taps = case
    dy, x = inputs(case, 3)
    nbytes = ws_bytes(*case)
    ref = run_wgrad(dy, x, taps)
    ws = torch.full((nbytes // 4,), float("nan"), device="cuda").view(torch.uint8)
    nan_ws = run_wgrad(dy, x, taps, ws=ws)
    again = run_wgrad(dy, x, taps)
    assert torch.isfinite(ref).all()
    assert torch.equal(ref.view(torch.int32), nan_ws.view(torch.int32))
    assert torch.equal(ref.view(torch.int32), again.view(torch.int32))


# ---- ConvFn --------------------------------------------------------------------------------------------------------------------
def rel_err(got, want):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    return float((got - want).abs().max() / (want.abs().max() + 1e-12))


@pytest.mark.parametrize("shape", [(3, 70, 256, 1024, 9, 1), (2, 133, 384, 384, 1, 0), (4, 41, 80, 256, 5, 0), (2, 50, 256, 256, 3, 1)])
def test_conv_fn_tf32_gradients(shape):
    B, L, K, N, taps, act = shape
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn(B, L, K, generator=g); w = torch.randn(N, K, taps, generator=g) / math.sqrt(K * taps); b = torch.randn(N, generator=g)
    gy = torch.randn(B, L, N, generator=g)
    xc, wc, bc = (t.cuda().requires_grad_() for t in (x, w, b))
    out = T.ConvFn.apply(xc, wc, bc, act, None, _lib.MATH_TF32)
    out.backward(gy.cuda())
    # float64 reference; behind the ReLU it back-propagates through this path's own mask (out > 0): tf32 rounding moves
    # pre-activations near zero across it, and a flipped mask element is a difference in the forward, not in the gradients
    xr, wr, br = (t.double().requires_grad_() for t in (x, w, b))
    y = torch.nn.functional.conv1d(xr.transpose(1, 2), wr, br, padding=(taps - 1) // 2).transpose(1, 2)
    gref = gy.double() * (out.detach().cpu() > 0).double() if act else gy.double()
    y.backward(gref)
    y = torch.relu(y) if act else y
    errs = [rel_err(out, y), rel_err(xc.grad, xr.grad), rel_err(wc.grad, wr.grad), rel_err(bc.grad, br.grad)]
    print(shape, "out / dx / dw / db:", ["%.2e" % e for e in errs])
    assert errs[0] < 5e-3 and errs[1] < 5e-3 and errs[2] < 2e-3 and errs[3] < 1e-5, errs
    # and it is not the fp32 path
    out32 = T.ConvFn.apply(xc.detach(), wc.detach(), bc.detach(), act, None)
    assert not torch.equal(out, out32)


# ---- the model -------------------------------------------------------------------------------------------------------------------
class _Recorded(T.MaskSource):
    """The reference's masks in call order, permuted to this path's layout where it drops a [B, C, time] tensor."""

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


def _golden_step(weights, golden, ragged, train_precision, record_shapes=None):
    g = golden("train_step_ragged" if ragged else "train_step")
    if ragged:
        bt = make_batch(3, 23, 181, seed=17, ilens=[23, 17, 9], olens=[181, 140, 66])
    else:
        bt = make_batch(2, 20, 150, seed=16)
    gen = torch.Generator().manual_seed(5)
    recorded = [torch.rand(shape, generator=gen) >= p for shape, p in zip(json.loads(str(g["mask_shapes"])), g["mask_rates"].tolist())]
    m = FeedForwardTransformer(68, 80, load_hp(), precision="fp32", train_precision=train_precision)
    m.load_state_dict(weights, strict=True)
    m = m.cuda().train()
    m.dropout_masks = _Recorded(recorded)
    if record_shapes is not None:
        apply = T.ConvFn.apply

        def recording(x, w, *rest):     # (bias, act, resid[, math])
            record_shapes.add((w.shape[0], w.shape[1], w.shape[2] if w.dim() == 3 else 1, rest[3] if len(rest) > 3 else None))
            return apply(x, w, *rest)
        T.ConvFn.apply = recording
    try:
        loss, rep = m(*[bt[k].cuda() for k in KEYS])
    finally:
        if record_shapes is not None:
            del T.ConvFn.apply          # back to torch.autograd.Function.apply
    loss.backward()
    torch.cuda.synchronize()
    assert not m.dropout_masks.recorded
    return g, m, loss, rep


# Gates from the first H100 run (DESIGN.md §10), at most 3x the observed worst of the two batches: loss 5.5e-7, report
# 3.3e-4, gradients 9.8e-2 (postnet.postnet.4.0.weight; relative to the reference's largest element), positional-encoding
# alpha 0.35, key bias 2.2e-7 (relative to the key weight's), BatchNorm buffers 4.4e-4 (relative to the buffer's largest)
LOSS_GATE, REPORT_GATE, GRAD_GATE, ALPHA_GATE, KBIAS_GATE, BUF_GATE = 1.5e-6, 1e-3, 0.25, 1.0, 6e-7, 1.2e-3


@pytest.mark.parametrize("ragged", [False, True])
def test_tf32_train_step_matches_reference_autograd(weights, golden, ragged):
    shapes = set()
    g, m, loss, rep = _golden_step(weights, golden, ragged, "tf32", record_shapes=shapes)
    assert {s[:3] for s in shapes} <= set(TRAIN_SHAPES), shapes - set(TRAIN_SHAPES)
    assert {s[3] for s in shapes} == {_lib.MATH_TF32}, "every ConvFn of the step ran in tf32"
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
            # softmax ignores a per-query constant: the key bias's gradient is exactly zero, the reference's and this
            # path's are rounding noise; bounded against the same layer's key-weight gradient instead
            kbias = max(kbias, err / float(g["gmax/" + name.replace(".bias", ".weight")]))
            continue
        errs[name] = err / (scale + 1e-12)
    # the positional-encoding scales' gradients are single sums of dy . pe over every element, mostly cancelling
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

    # the mode switched: the fp32 step's gradients differ
    _, m32, _, _ = _golden_step(weights, golden, ragged, "fp32")
    g32 = dict(m32.named_parameters())
    assert any(p.grad is not None and not torch.equal(p.grad, g32[n].grad) for n, p in m.named_parameters())


def test_tf32_optimizer_step_through_the_reference_training_recipe(weights):
    m = FeedForwardTransformer(68, 80, load_hp(), precision="fp32", train_precision="tf32")
    m.load_state_dict(weights, strict=True)
    m = m.cuda()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    bt = make_batch(2, 20, 150, seed=21)
    args = [bt[k].cuda() for k in KEYS]
    m.eval()
    with torch.no_grad():
        l0, _ = m(*args)
    m.train()
    losses = []
    for _ in range(3):
        loss, _ = m(*args)
        loss.backward()
        gn = torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0)
        assert math.isfinite(float(gn))
        opt.step(); opt.zero_grad()
        losses.append(float(loss))
    m.eval()
    with torch.no_grad():
        l1, _ = m(*args)
    assert float(l1) < float(l0), (float(l0), float(l1), losses)


@pytest.mark.parametrize("precision", ["3xf16", "tf32", "fp32"])
def test_eval_is_unaffected_by_the_train_mode(weights, precision):
    bt = make_batch(3, 23, 181, seed=17, ilens=[23, 17, 9], olens=[181, 140, 66])
    outs = []
    for tp in ("fp32", "tf32"):
        m = FeedForwardTransformer(68, 80, load_hp(), precision=precision, train_precision=tp)
        m.load_state_dict(weights, strict=True)
        m = m.cuda().eval()
        with torch.no_grad():
            outs.append(m._forward(*[bt[k].cuda() for k in ("xs", "ilens", "olens", "ds", "es", "ps")], is_inference=False))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
