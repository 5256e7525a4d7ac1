"""The fp32 train kernels (csrc/train.cu) one entry point at a time, against float64, at the train bench's shapes and at
the edges of their launch geometry (tests/_train_plan.py).

* every entry is called through the C ABI (and through its torch.autograd.Function where there is one);
* references are float64 restatements of the reference ops (F.layer_norm, F.batch_norm, conv1d as shifted matmuls,
  masked softmax, ...), autograd for the backward passes, on the GPU for the large shapes;
* element-wise entries must equal the fp32 torch expression in the same operation order bit for bit;
* reductions are gated on max |err| / sum |terms| (the sum of the absolute values of everything that was added, including
  the caller's starting value where the entry accumulates).  Each gate is 3x the worst value of the first H100 runs
  (OBSERVED below), and each case is also held to its a-priori ceiling `n_chain * 2^-24` from the plan, whichever is
  tighter;
* every output sits between sentinel guard bands; accumulated outputs start from seeded nonzero values; inputs the kernel
  must not read for its values (padding) hold NaN or large finite garbage.

The worst ratio per entry is printed at the end of the module (`-s`).  Needs an H100: run with `-m gpu`."""
import ast
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _train_plan as P
from _wgrad_plan import TRAIN_SHAPES
from fastspeech2_b200 import _lib
from fastspeech2_b200 import train as T

pytestmark = pytest.mark.gpu
GUARD = 64
SENT = 12345.5
DEV = "cuda"
NAN = float("nan")

# Worst max |err| / sum |terms| per entry over the first H100 runs (NVIDIA H100 80GB HBM3, power limit 700 W, max SM
# clock 1980 MHz; the atomics' order varies from run to run).  Each gate is 3x that; a case is also held to its ceiling
# n_chain * 2^-24 from tests/_train_plan.py when that is tighter.
OBSERVED = {
    "colsum": 1.41e-07, "conv_forward": 4.36e-07, "conv_dgrad": 5.25e-07, "conv_wgrad": 3.74e-07,
    "conv_wgrad.dbias": 8.35e-08, "layernorm.dx": 2.18e-07, "layernorm.dgamma": 1.23e-07, "layernorm.dbeta": 1.45e-07,
    "batchnorm.stats": 5.92e-08, "batchnorm.y": 2.09e-07, "batchnorm.running": 1.32e-07, "batchnorm.dx": 1.96e-07,
    "batchnorm.dgamma": 1.22e-07, "batchnorm.dbeta": 9.61e-08, "bgemm": 2.89e-07, "softmax.p": 2.41e-07,
    "softmax.ds": 2.67e-07, "attention": 1.40e-06, "embed.dtable": 2.05e-07, "embed.dalpha": 1.95e-09,
    "onehot.dW": 2.48e-07, "length_regulator": 2.04e-07, "rowdot.y": 4.74e-08, "rowdot.dw": 6.40e-08,
    "rowdot.dbias": 3.24e-08, "loss.values": 5.21e-08, "loss.grads": 1.64e-07,
}
GATES = {k: 3 * v for k, v in OBSERVED.items()}
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst max |err| / sum |terms| per entry (gate; the smallest ceiling n_chain * 2^-24 among its cases):")
    for k in sorted(WORST):
        v, g, c = WORST[k]
        print(f"  {k:20s} {v:.3e}   gate {g:.1e}   ceiling {c:.1e}")


def lib():
    return _lib.load()


def call(name, *args):
    """One C-ABI entry on the current stream; raises with the library's message on an error code."""
    _lib.check(getattr(lib(), name)(*args, torch.cuda.current_stream().cuda_stream), name)


def rnd(shape, seed, scale=1.0, shift=0.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(shape, generator=g, device=DEV) * scale + shift


class Guarded:
    """n elements with GUARD sentinel elements on each side."""

    def __init__(self, n, fill=None, dtype=torch.float32, sentinel=SENT):
        self.n, self.sentinel = n, sentinel
        self.buf = torch.full((n + 2 * GUARD,), sentinel, dtype=dtype, device=DEV)
        self.v = self.buf[GUARD:GUARD + n]
        if fill is not None:
            self.v.copy_(fill.reshape(-1))

    @property
    def ptr(self):
        return self.v.data_ptr()

    def intact(self):
        b = self.buf
        return bool((b[:GUARD] == self.sentinel).all()) and bool((b[GUARD + self.n:] == self.sentinel).all())


def ratio(got, want, terms):
    """max |got - want| / terms; where terms is 0 the result must be exact."""
    got, want, terms = (t.detach().double().reshape(-1) for t in (got, want, terms))
    err = (got - want).abs()
    zero = terms == 0
    assert not bool(err[zero].ne(0).any()), "nonzero (or NaN) error where every term is 0"
    if bool(torch.isnan(err).any()):
        return math.inf
    nz = ~zero
    return float((err[nz] / terms[nz]).max()) if bool(nz.any()) else 0.0


def gate(entry, r, chain):
    """Hold r to min(the entry's gate, this case's ceiling chain * 2^-24) and record the worst."""
    ceiling = chain * P.U24
    g = min(GATES[entry], ceiling)
    v, _, c = WORST.get(entry, (0.0, 0.0, math.inf))
    WORST[entry] = (max(v, r), GATES[entry], min(c, ceiling))
    assert r <= g, f"{entry}: max |err| / sum |terms| = {r:.3e} > {g:.2e} (gate {GATES[entry]:.1e}, ceiling {ceiling:.1e})"


def bits(t):
    return t.contiguous().view(torch.int32)


def free():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


# ---- dropout mask: a numpy Philox4x32-10 restatement ---------------------------------------------------------------------
M32 = np.uint64(0xFFFFFFFF)


def philox4x32(c0, c1, k0, k1):
    """Philox4x32-10 (common.cuh) on counters (c0, c1, 0, 0), key (k0, k1); 32-bit words held in uint64 arrays."""
    x0, x1 = c0 & M32, c1 & M32
    x2 = np.zeros_like(x0)
    x3 = np.zeros_like(x0)
    k0, k1 = np.uint64(k0), np.uint64(k1)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * x0
        p1 = np.uint64(0xCD9E8D57) * x2
        x0, x1, x2, x3 = (p1 >> np.uint64(32)) ^ x1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ x3 ^ k1, p0 & M32
        k0 = (k0 + np.uint64(0x9E3779B9)) & M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & M32
    return x0, x1, x2, x3


def ref_mask(n, p, seed, offset):
    """Byte i: word i % 4 of quad i / 4, quad q drawn at counter offset + q (carrying into the high word); kept iff
    (w >> 8) * 2^-24 >= p in fp32."""
    q = np.arange((n + 3) // 4, dtype=np.uint64)
    c = np.uint64(offset) + q
    words = philox4x32(c & M32, c >> np.uint64(32), seed & 0xFFFFFFFF, seed >> 32)
    w = np.stack(words, 1).reshape(-1)[:n]
    u = (w >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)
    return (u >= np.float32(p)).astype(np.uint8)


MASK_SEEDS = [1234, (0x9E3779B9 << 32) | 0x7F4A7C15]     # the second has its high word set


def test_dropout_mask_matches_a_philox_restatement():
    """fs2_dropout_mask bit for bit; offsets 2^32 - 2 (the counter carries inside one call) and 2^32 + 5 pin the high word."""
    for seed in MASK_SEEDS:
        for n in (1, 2, 3, 4, 5, 4097):
            for off in (0, 7, 2 ** 32 - 2, 2 ** 32 + 5):
                for p in (0.0, 0.2, 0.5, 0.9):
                    m = Guarded(n, dtype=torch.uint8, sentinel=0xAB)
                    call("fs2_dropout_mask", m.ptr, n, p, seed, off)
                    torch.cuda.synchronize()
                    assert m.intact(), (seed, n, off, p)
                    assert np.array_equal(m.v.cpu().numpy(), ref_mask(n, p, seed, off)), (seed, n, off, p)
    # keep rate sanity on a large draw
    assert abs(ref_mask(1 << 16, 0.2, 99, 0).mean() - 0.8) < 0.01


def test_mask_source_gives_successive_calls_disjoint_counters():
    seed = MASK_SEEDS[1]
    src = T.MaskSource(seed=seed)
    m1 = src.next((5, 7, 3), 0.2, torch.device(DEV))
    m2 = src.next((4097,), 0.2, torch.device(DEV))
    assert np.array_equal(m1.reshape(-1).cpu().numpy(), ref_mask(105, 0.2, seed, 0))
    assert np.array_equal(m2.cpu().numpy(), ref_mask(4097, 0.2, seed, 27))        # ceil(105 / 4) quads later
    assert src.offset == 27 + 1025


# ---- element-wise entries: bit for bit -----------------------------------------------------------------------------------------
N_EW = 1_000_003      # past the grid cap (1056 CTAs x 256), not a multiple of the block


def _ew_inputs(seed):
    x = rnd(N_EW, seed)
    x[::97] = 0.0
    x[1::97] = -0.0
    return x


def test_dropout_apply_bit_for_bit():
    """out = mask ? x * float(1 / (1 - p)) : +0; x at dropped positions is NaN and must not reach out."""
    x = _ew_inputs(1)
    keep = torch.rand(N_EW, generator=torch.Generator(device=DEV).manual_seed(2), device=DEV) >= 0.3
    mask = keep.to(torch.uint8)
    xn = torch.where(keep, x, torch.full_like(x, NAN))
    for p in (0.0, 0.2, 0.5, 0.9):
        scale = torch.tensor(np.float32(1.0) / (np.float32(1.0) - np.float32(p)), device=DEV)
        want = torch.where(keep, x * scale, torch.zeros_like(x))
        out = Guarded(N_EW)
        call("fs2_dropout_apply", xn.data_ptr(), mask.data_ptr(), p, out.ptr, N_EW)
        torch.cuda.synchronize()
        assert out.intact() and torch.equal(bits(out.v), bits(want)), p
    # DropoutFn: forward and backward are the same map
    xr = x.clone().requires_grad_()
    y = T.DropoutFn.apply(xr, mask, 0.2)
    gy = rnd(N_EW, 3)
    y.backward(gy)
    scale = torch.tensor(np.float32(1.0) / np.float32(0.8), device=DEV)
    assert torch.equal(bits(y), bits(torch.where(keep, x * scale, torch.zeros_like(x))))
    assert torch.equal(bits(xr.grad), bits(torch.where(keep, gy * scale, torch.zeros_like(x))))


def test_relu_and_add_bit_for_bit():
    """fs2_relu = fmaxf(x, 0): equal to clamp_min(x, 0) as values; the sign of a zero result is fmaxf's choice, so bits
    are compared where the result is nonzero.  fs2_add = a + b bit for bit (ReluFn / AddFn too)."""
    x = _ew_inputs(4)
    y = Guarded(N_EW)
    call("fs2_relu", x.data_ptr(), y.ptr, N_EW)
    want = x.clamp_min(0.0)
    torch.cuda.synchronize()
    assert y.intact() and torch.equal(y.v, want)
    nz = want != 0
    assert torch.equal(bits(y.v[nz]), bits(want[nz]))
    b = rnd(N_EW, 5)
    s = Guarded(N_EW)
    call("fs2_add", x.data_ptr(), b.data_ptr(), s.ptr, N_EW)
    torch.cuda.synchronize()
    assert s.intact() and torch.equal(bits(s.v), bits(x + b))
    xr = x.clone().requires_grad_()
    r = T.ReluFn.apply(xr)
    gy = rnd(N_EW, 6)
    r.backward(gy)
    assert torch.equal(r, want) and torch.equal(bits(xr.grad), bits(torch.where(r > 0, gy, torch.zeros_like(gy))))
    assert torch.equal(bits(T.AddFn.apply(x, b)), bits(x + b))


def test_act_backward_bit_for_bit():
    """dx = dy (none), y > 0 ? dy : 0 (relu, y exactly 0 included), dy * (1 - y^2) (tanh).  nvcc contracts 1 - y*y into
    one FMA, so the tanh restatement rounds 1 - y^2 once: |y| is kept in [1/8, 1] or 0, where 1 - y^2 is exact in float64."""
    dy = rnd(N_EW, 7)
    yr = torch.where(rnd(N_EW, 8) > 0, rnd(N_EW, 9), torch.zeros(N_EW, device=DEV))
    yr[::101] = 0.0
    yr[1::101] = -0.0
    g = torch.Generator(device=DEV).manual_seed(10)
    mag = 0.125 + 0.875 * torch.rand(N_EW, generator=g, device=DEV)
    mag[::13] = 1.0
    mag[1::13] = 1.0 - 2.0 ** -24
    mag[2::13] = 1.0 - 2.0 ** -20
    mag[3::13] = 0.0
    yt = mag * torch.where(rnd(N_EW, 11) > 0, 1.0, -1.0)
    cases = [(T.ACT_NONE, yr, dy), (T.ACT_RELU, yr, torch.where(yr > 0, dy, torch.zeros_like(dy))),
             (T.ACT_TANH, yt, (dy.double() * (1.0 - yt.double() ** 2).float().double()).float())]
    for act, y, want in cases:
        dx = Guarded(N_EW)
        call("fs2_act_backward", dy.data_ptr(), y.data_ptr(), act, dx.ptr, N_EW)
        torch.cuda.synchronize()
        assert dx.intact() and torch.equal(bits(dx.v), bits(want)), act


# ---- column sums ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", P.COLSUM_CS)
@pytest.mark.parametrize("rows", P.COLSUM_ROWS)
def test_colsum(rows, C):
    """out += sum_r x[r]: against float64, from seeded starting values."""
    x = rnd((rows, C), rows * 7 + C)
    init = rnd(C, C + 1)
    out = Guarded(C, fill=init)
    call("fs2_colsum", x.data_ptr(), rows, C, out.ptr)
    want = init.double() + x.double().sum(0)
    terms = init.double().abs() + x.double().abs().sum(0)
    torch.cuda.synchronize()
    assert out.intact()
    gate("colsum", ratio(out.v, want, terms), P.colsum(rows, C)["chain"])


# ---- convolution (fp32) ----------------------------------------------------------------------------------------------------------
def conv64(x, w):
    """float64 "same" conv1d of x [B, L, K] with w [N, K, taps] as taps shifted matmuls -> [B, L, N]."""
    B, L, K = x.shape
    N, _, taps = w.shape
    pad = (taps - 1) // 2
    xp = F.pad(x, (0, 0, pad, pad))
    y = torch.zeros(B, L, N, dtype=torch.float64, device=x.device)
    for j in range(taps):
        y += xp[:, j:j + L] @ w[:, :, j].T
    return y


def dgrad64(dy, w):
    """float64 adjoint of conv64 in x: dx[b, t] = sum_j dy[b, t - j + pad] w[:, :, j]."""
    B, L, N = dy.shape
    taps = w.shape[2]
    pad = (taps - 1) // 2
    dp = F.pad(dy, (0, 0, pad, pad))
    dx = torch.zeros(B, L, w.shape[1], dtype=torch.float64, device=dy.device)
    for j in range(taps):
        dx += dp[:, taps - 1 - j:taps - 1 - j + L] @ w[:, :, j]
    return dx


def wgrad64(dy, x, taps):
    B, L, N = dy.shape
    pad = (taps - 1) // 2
    xp = F.pad(x, (0, 0, pad, pad))
    w = torch.empty(N, x.shape[2], taps, dtype=torch.float64, device=dy.device)
    for j in range(taps):
        w[:, :, j] = dy.reshape(-1, N).T @ xp[:, j:j + L].reshape(-1, x.shape[2])
    return w


CONV_CASES = P.conv_cases(TRAIN_SHAPES)


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "B%d_L%d_N%d_K%d_t%d" % c)
def test_conv_forward_dgrad_wgrad(case):
    """fs2_conv_forward (+ bias), fs2_conv_dgrad and fs2_conv_wgrad (+= from seeded values, with the bias gradient) against
    float64; dgrad is the adjoint of forward; the _ex entries in FS2_MATH_FP32 are the same calls, bit for bit."""
    B, L, N, K, taps = case
    s = sum(case)
    x = rnd((B, L, K), s, 0.5, 0.1)
    w = rnd((N, K, taps), s + 1, 1.0 / math.sqrt(K * taps))
    bias = rnd(N, s + 2)
    dy = rnd((B, L, N), s + 3)
    scratch = torch.empty(N * K * taps, device=DEV)
    plan = P.wgrad(B, L, N, K, taps)
    x64, w64, dy64 = x.double(), w.double(), dy.double()

    out = Guarded(B * L * N)
    call("fs2_conv_forward", x.data_ptr(), B, L, K, w.data_ptr(), bias.data_ptr(), N, taps, T.ACT_NONE, None, out.ptr, scratch.data_ptr())
    want = conv64(x64, w64) + bias.double()
    terms = conv64(x64.abs(), w64.abs()) + bias.double().abs()
    torch.cuda.synchronize()
    assert out.intact()
    gate("conv_forward", ratio(out.v, want, terms), plan["fwd_chain"])
    out_ex = torch.empty(B * L * N, device=DEV)
    call("fs2_conv_forward_ex", x.data_ptr(), B, L, K, w.data_ptr(), bias.data_ptr(), N, taps, T.ACT_NONE, None, out_ex.data_ptr(),
         scratch.data_ptr(), _lib.MATH_FP32)
    assert torch.equal(bits(out_ex), bits(out.v))
    del want, terms

    dx = Guarded(B * L * K)
    call("fs2_conv_dgrad", dy.data_ptr(), B, L, N, w.data_ptr(), K, taps, dx.ptr, scratch.data_ptr())
    want = dgrad64(dy64, w64)
    terms = dgrad64(dy64.abs(), w64.abs())
    torch.cuda.synchronize()
    assert dx.intact()
    gate("conv_dgrad", ratio(dx.v, want, terms), plan["dgrad_chain"])
    dx_ex = torch.empty(B * L * K, device=DEV)
    call("fs2_conv_dgrad_ex", dy.data_ptr(), B, L, N, w.data_ptr(), K, taps, dx_ex.data_ptr(), scratch.data_ptr(), _lib.MATH_FP32)
    assert torch.equal(bits(dx_ex), bits(dx.v))
    del want, terms

    # <conv(x), dy> = <x, dgrad(dy)> on the fp32 results (no bias)
    y0 = torch.empty(B * L * N, device=DEV)
    call("fs2_conv_forward", x.data_ptr(), B, L, K, w.data_ptr(), None, N, taps, T.ACT_NONE, None, y0.data_ptr(), scratch.data_ptr())
    lhs = float((y0.double() * dy64.reshape(-1)).sum())
    rhs = float((x64.reshape(-1) * dx.v.double()).sum())
    scale = float((conv64(x64.abs(), w64.abs()) * dy64.abs()).sum())
    assert abs(lhs - rhs) <= (plan["fwd_chain"] + plan["dgrad_chain"]) * P.U24 * scale, (lhs, rhs, scale)
    del y0, dx

    _check_wgrad(dy, x, taps, plan)
    free()


def _check_wgrad(dy, x, taps, plan):
    B, L, N = dy.shape
    K = x.shape[2]
    n = N * K * taps
    init = rnd(n, n + 5)
    binit = rnd(N, N + 6)
    dw = Guarded(n, fill=init)
    db = Guarded(N, fill=binit)
    _lib.check(lib().fs2_conv_wgrad(dy.data_ptr(), x.data_ptr(), B, L, N, K, taps, dw.ptr, db.ptr,
                                    torch.cuda.current_stream().cuda_stream), "fs2_conv_wgrad")
    dy64, x64 = dy.double(), x.double()
    want = init.double().reshape(N, K, taps) + wgrad64(dy64, x64, taps)
    terms = init.double().abs().reshape(N, K, taps) + wgrad64(dy64.abs(), x64.abs(), taps)
    torch.cuda.synchronize()
    assert dw.intact() and db.intact()
    gate("conv_wgrad", ratio(dw.v, want, terms), plan["chain"])
    dsum = dy64.reshape(-1, N)
    gate("conv_wgrad.dbias", ratio(db.v, binit.double() + dsum.sum(0), binit.double().abs() + dsum.abs().sum(0)),
         P.colsum(B * L, N)["chain"])


@pytest.mark.parametrize("case", P.WGRAD_TAIL_CASES, ids=lambda c: "B%d_L%d_N%d_K%d_t%d" % c)
def test_conv_wgrad_tails(case):
    """N, K tails of 1 and 65 of the 64 x 64 weight-gradient tiles (shapes only fs2_conv_wgrad accepts)."""
    B, L, N, K, taps = case
    _check_wgrad(rnd((B, L, N), sum(case)), rnd((B, L, K), sum(case) + 1, 0.5, 0.1), taps, P.wgrad(*case))


def test_conv_fn_fp32_matches_the_entries():
    """ConvFn (fp32) at a c2 shape: the same numbers as the entries, gated the same way."""
    B, L, N, K, taps = 64, 100, 256, 256, 3
    x = rnd((B, L, K), 1, 0.5, 0.1).requires_grad_()
    w = rnd((N, K, taps), 2, 1.0 / math.sqrt(K * taps)).requires_grad_()
    b = rnd(N, 3).requires_grad_()
    gy = rnd((B, L, N), 4)
    out = T.ConvFn.apply(x, w, b, T.ACT_NONE, None)
    out.backward(gy)
    plan = P.wgrad(B, L, N, K, taps)
    x64, w64, g64 = x.detach().double(), w.detach().double(), gy.double()
    gate("conv_forward", ratio(out, conv64(x64, w64) + b.detach().double(), conv64(x64.abs(), w64.abs()) + b.detach().double().abs()),
         plan["fwd_chain"])
    gate("conv_dgrad", ratio(x.grad, dgrad64(g64, w64), dgrad64(g64.abs(), w64.abs())), plan["dgrad_chain"])
    gate("conv_wgrad", ratio(w.grad, wgrad64(g64, x64, taps), wgrad64(g64.abs(), x64.abs(), taps)), plan["chain"])


# ---- LayerNorm backward -------------------------------------------------------------------------------------------------------------
LN_CASES = [(r, C, 1e-5) for C in P.LN_CS for r in P.LN_ROWS] + [(r, 256, 1e-12) for r in P.LN_ROWS]


def _ln_input(rows, C, seed):
    x = rnd((rows, C), seed, 2.0, 0.3)
    x[0] = 1.5                                   # constant rows (variance 0); dyadic, so the fp32 mean is exact
    if rows > 2:
        x[2] = -0.75
    if rows > 1:
        x[1] = rnd(C, seed + 1, 1.0, 1e3)        # mean / std = 1e3
        x[-1] = rnd(C, seed + 2, 1.0, -1e3)
    return x


@pytest.mark.parametrize("case", LN_CASES, ids=lambda c: "rows%d_C%d_eps%g" % c)
def test_layernorm_backward(case):
    """fs2_layernorm_backward against F.layer_norm's float64 autograd.  Centring a row in fp32 leaves xhat an absolute
    error of up to kappa u, kappa = |mean| rstd (the mean's rounding, scaled), on top of its relative error.  dx depends
    on xhat through xhat mean(g xhat), so kappa enters its terms once, as the first-order perturbation of that product:
    rstd (|g| + mean|g| + |xhat| mean|g xhat| + kappa (mean|g xhat| + |xhat| mean|g|)) with g = dy gamma.  dgamma:
    sum |dy| (|xhat| + kappa); dbeta: sum |dy|; both plus the starting value.  A constant row at C = 384 shows why kappa
    is there: its fp32 mean, a product with fp32(1 / 384), is an ulp off, so its xhat is kappa u rather than 0.  On the
    mean / std = 1e3 rows a variance off by a few per cent (one-pass E[x^2] - mean^2 in fp32) fails the dx gate; on the
    constant rows at eps = 1e-12 so does a kernel that drops eps."""
    rows, C, eps = case
    x = _ln_input(rows, C, rows + C)
    dy = rnd((rows, C), rows + C + 3)
    gamma = rnd(C, C, 0.2, 1.0)
    ig, ib = rnd(C, 11), rnd(C, 12)
    dx, dg, db = Guarded(rows * C), Guarded(C, fill=ig), Guarded(C, fill=ib)
    call("fs2_layernorm_backward", x.data_ptr(), dy.data_ptr(), gamma.data_ptr(), eps, rows, C, dx.ptr, dg.ptr, db.ptr)

    e = float(np.float32(eps))
    x64 = x.double().requires_grad_()
    g64 = gamma.double().requires_grad_()
    b64 = torch.zeros(C, dtype=torch.float64, device=DEV, requires_grad=True)
    dy64 = dy.double()
    F.layer_norm(x64, (C,), g64, b64, e).backward(dy64)
    with torch.no_grad():
        xd = x.double()
        mean, var = xd.mean(-1, keepdim=True), xd.var(-1, unbiased=False, keepdim=True)
        rstd = 1.0 / torch.sqrt(var + e)
        xhat = (xd - mean) * rstd
        kappa = mean.abs() * rstd
        ax = xhat.abs()
        gg = (dy64 * gamma.double()).abs()
        m_g, m_gx = gg.mean(-1, keepdim=True), (gg * ax).mean(-1, keepdim=True)
        t_dx = rstd * (gg + m_g + ax * m_gx + kappa * (m_gx + ax * m_g))
        t_dg = ig.double().abs() + (dy64.abs() * (ax + kappa)).sum(0)
        t_db = ib.double().abs() + dy64.abs().sum(0)
    torch.cuda.synchronize()
    assert dx.intact() and dg.intact() and db.intact()
    ch = P.layernorm_chain(rows, C)
    gate("layernorm.dx", ratio(dx.v, x64.grad, t_dx), ch["dx"])
    gate("layernorm.dgamma", ratio(dg.v, ig.double() + g64.grad, t_dg), ch["dgamma"])
    gate("layernorm.dbeta", ratio(db.v, ib.double() + b64.grad, t_db), ch["dgamma"])
    if rows == 4225:
        # LayerNormFn: the same entry behind autograd (zero starting values)
        xr, gr = x.clone().requires_grad_(), gamma.clone().requires_grad_()
        br = torch.zeros(C, device=DEV, requires_grad=True)
        T.LayerNormFn.apply(xr, gr, br, eps).backward(dy)
        gate("layernorm.dx", ratio(xr.grad, x64.grad, t_dx), ch["dx"])
        gate("layernorm.dgamma", ratio(gr.grad, g64.grad, t_dg - ig.double().abs()), ch["dgamma"])
        gate("layernorm.dbeta", ratio(br.grad, b64.grad, t_db - ib.double().abs()), ch["dgamma"])
    free()


# ---- BatchNorm (train) --------------------------------------------------------------------------------------------------------------
BN_CASES = [(r, C) for C in P.BN_CS for r in P.BN_ROWS]


@pytest.mark.parametrize("act", [T.ACT_NONE, T.ACT_TANH], ids=["none", "tanh"])
@pytest.mark.parametrize("case", BN_CASES, ids=lambda c: "rows%d_C%d" % c)
def test_batchnorm_train_and_backward(case, act):
    """fs2_batchnorm_train (statistics, output, running statistics with the unbiased variance at momentum 0.1) and
    fs2_batchnorm_backward against F.batch_norm's float64 autograd (BatchNorm1d in train mode).  Channel 0 has
    mean / std = 1e3: the statistics are one-pass E[x^2] - mean^2 in double, exact to far below fp32 there; the mean's
    rounding to fp32 leaves xhat an absolute error of kappa u, kappa = |mean| rstd: y and dgamma use |xhat| + kappa in
    place of |xhat|, and dx, which depends on xhat through xhat sum(dy xhat), takes kappa once, as the first-order
    perturbation of that product (as for LayerNorm)."""
    rows, C = case
    s = rows + C + act
    x = rnd((rows, C), s, 1.5, 0.2)
    x[:, 0] = rnd(rows, s + 1, 1.0, 1e3)
    gamma, beta = rnd(C, s + 2, 0.1, 1.0), rnd(C, s + 3)
    rm0, rv0 = rnd(C, s + 4), rnd(C, s + 5).abs() + 0.5
    rm, rv = rm0.clone(), rv0.clone()
    eps, mom = 1e-5, 0.1
    stats = Guarded(2 * C)
    y = Guarded(rows * C)
    scratch = torch.empty(4 * C, dtype=torch.float64, device=DEV)
    call("fs2_batchnorm_train", x.data_ptr(), rows, C, gamma.data_ptr(), beta.data_ptr(), eps, mom, act, rm.data_ptr(), rv.data_ptr(),
         stats.ptr, y.ptr, scratch.data_ptr())
    e, m = float(np.float32(eps)), float(np.float32(mom))
    x64 = x.double().requires_grad_()
    g64, b64 = gamma.double().requires_grad_(), beta.double().requires_grad_()
    rm64, rv64 = rm0.double(), rv0.double()
    z = F.batch_norm(x64, rm64, rv64, g64, b64, training=True, momentum=m, eps=e)
    with torch.no_grad():
        xd = x.double()
        mean, var = xd.mean(0), xd.var(0, unbiased=False)
        rstd = 1.0 / torch.sqrt(var + e)
        xhat = (xd - mean) * rstd
        kappa = mean.abs() * rstd
        a = xhat.abs() + kappa
        t_z = gamma.double().abs() * a + beta.double().abs()
        zd = z.detach()
        want_y = torch.tanh(zd) if act == T.ACT_TANH else zd
        t_y = (1 - want_y ** 2) * t_z + want_y.abs() if act == T.ACT_TANH else t_z
    torch.cuda.synchronize()
    assert stats.intact() and y.intact()
    ch = P.bn(rows)["chain"]
    gate("batchnorm.stats", ratio(stats.v[:C], mean, xd.abs().mean(0)), ch)
    gate("batchnorm.stats", ratio(stats.v[C:], var, var), ch)
    gate("batchnorm.y", ratio(y.v, want_y, t_y), ch)
    gate("batchnorm.running", ratio(rm, rm64, (1 - m) * rm0.double().abs() + m * mean.abs()), ch)
    gate("batchnorm.running", ratio(rv, rv64, (1 - m) * rv0.double().abs() + m * var * rows / max(rows - 1, 1)), ch)

    dy = rnd((rows, C), s + 6)
    ig, ib = rnd(C, s + 7), rnd(C, s + 8)
    dx, dg, db = Guarded(rows * C), Guarded(C, fill=ig), Guarded(C, fill=ib)
    call("fs2_batchnorm_backward", x.data_ptr(), dy.data_ptr(), stats.ptr, gamma.data_ptr(), eps, rows, C, dx.ptr, dg.ptr, db.ptr,
         scratch.data_ptr())
    dy64 = dy.double()
    z.backward(dy64)
    with torch.no_grad():
        ad = dy64.abs()
        m_d, m_dx = ad.sum(0) / rows, (ad * xhat.abs()).sum(0) / rows
        t_dx = gamma.double().abs() * rstd * (ad + m_d + xhat.abs() * m_dx + kappa * (m_dx + xhat.abs() * m_d))
        t_dg = ig.double().abs() + (dy64.abs() * a).sum(0)
        t_db = ib.double().abs() + dy64.abs().sum(0)
    torch.cuda.synchronize()
    assert dx.intact() and dg.intact() and db.intact()
    gate("batchnorm.dx", ratio(dx.v, x64.grad, t_dx), ch)
    gate("batchnorm.dgamma", ratio(dg.v, ig.double() + g64.grad, t_dg), ch)
    gate("batchnorm.dbeta", ratio(db.v, ib.double() + b64.grad, t_db), ch)
    if rows == 257 and C == 80:
        # BatchNormFn: fs2_act_backward then the entries above, behind autograd.  Two row blocks per channel and one
        # atomic per output onto zero, so the same inputs give the same bits.
        xr, gr, br = x.clone().requires_grad_(), gamma.clone().requires_grad_(), beta.clone().requires_grad_()
        rm2, rv2 = rm0.clone(), rv0.clone()
        yf = T.BatchNormFn.apply(xr, gr, br, rm2, rv2, eps, mom, act)
        assert torch.equal(yf.reshape(-1), y.v) and torch.equal(rm2, rm) and torch.equal(rv2, rv)
        yf.backward(dy)
        gin = torch.empty_like(dy)
        call("fs2_act_backward", dy.data_ptr(), y.ptr, act, gin.data_ptr(), rows * C)
        dx2, dg2, db2 = torch.empty_like(dy), torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
        call("fs2_batchnorm_backward", x.data_ptr(), gin.data_ptr(), stats.ptr, gamma.data_ptr(), eps, rows, C, dx2.data_ptr(), dg2.data_ptr(),
             db2.data_ptr(), scratch.data_ptr())
        assert torch.equal(xr.grad, dx2) and torch.equal(gr.grad, dg2) and torch.equal(br.grad, db2)
    free()


# ---- batched GEMM -------------------------------------------------------------------------------------------------------------------
def _layout(kind, Bt, h, rows, cols):
    """(base shape, (batch, head, row, col) strides) of an operand [rows, cols] per (b, h) in the layouts AttentionFn uses:
    'feat' rows of [Bt, rows, h*cols]; 'featT' its transpose; 'score' [Bt, h, rows, cols]; 'scoreT' its transpose.
    `extra` heads of columns are added to feat outputs by the caller."""
    if kind == "feat":
        return (Bt, rows, h * cols), (rows * h * cols, cols, h * cols, 1)
    if kind == "featT":
        return (Bt, cols, h * rows), (cols * h * rows, rows, 1, h * rows)
    if kind == "score":
        return (Bt, h, rows, cols), (h * rows * cols, rows * cols, cols, 1)
    return (Bt, h, cols, rows), (h * rows * cols, rows * cols, 1, rows)      # scoreT


# the six products of AttentionFn: (A, B, C) layouts
BGEMM_PATTERNS = {"q.kT": ("feat", "featT", "score"), "pd.v": ("score", "feat", "feat"), "pdT.dO": ("scoreT", "feat", "feat"),
                  "dO.vT": ("feat", "featT", "score"), "dS.k": ("score", "feat", "feat"), "dST.q": ("scoreT", "feat", "feat")}


@pytest.mark.parametrize("case", P.bgemm_cases(), ids=lambda c: "%s_M%d_N%d_K%d_h%d" % c)
def test_bgemm(case):
    """fs2_bgemm in AttentionFn's six stride patterns, alpha != 1; a feat output is written into a [B, M, (h+1) N] view
    whose last head's columns hold sentinels and must come back untouched."""
    pat, M, N, K, h = case
    Bt, alpha = 2, float(np.float32(0.37))         # the fp32 alpha the kernel multiplies by
    ka, kb, kc = BGEMM_PATTERNS[pat]
    sa, ta = _layout(ka, Bt, h, M, K)
    sb, tb = _layout(kb, Bt, h, K, N)
    s = M * 1000 + N * 10 + K
    a = rnd(sa, s)
    b = rnd(sb, s + 1)
    if kc == "feat":
        cshape, tc = (Bt, M, (h + 1) * N), (M * (h + 1) * N, N, (h + 1) * N, 1)
    else:
        cshape, tc = _layout(kc, Bt, h, M, N)
    nc = int(np.prod(cshape))
    c = Guarded(nc)
    call("fs2_bgemm", a.data_ptr(), *ta, b.data_ptr(), *tb, c.ptr, *tc, Bt, h, M, N, K, alpha)
    A = a.double().as_strided((Bt, h, M, K), ta)
    Bm = b.double().as_strided((Bt, h, K, N), tb)
    want = alpha * (A @ Bm)
    terms = alpha * (A.abs() @ Bm.abs())
    got = c.v.as_strided((Bt, h, M, N), tc)
    torch.cuda.synchronize()
    assert c.intact()
    if kc == "feat":
        assert bool((c.v.reshape(cshape)[:, :, h * N:] == SENT).all()), "another head's columns were written"
    gate("bgemm", ratio(got, want, terms), P.bgemm(M, N, K)["chain"])
    free()


# ---- attention softmax -------------------------------------------------------------------------------------------------------------
def _softmax_ref(s, lens, keep, dmask, heads):
    """float64 masked softmax (query and key < len), masked_fill 0, dropout; and its exp conditioning 1 + |s - max|."""
    B, L = lens.shape[0], s.shape[-1]
    valid = torch.arange(L, device=DEV)[None] < lens.clamp(max=L)[:, None]
    m = (valid[:, None, :] & valid[:, :, None])[:, None]                 # [B, 1, L, L]
    sd = s.double().masked_fill(~m, -math.inf)
    mx = sd.amax(-1, keepdim=True)
    p = torch.softmax(sd, -1).masked_fill(~m, 0.0)
    cond = 1.0 + (sd - mx).abs().masked_fill(~m, 0.0)
    pd = p if dmask is None else p * dmask.double() * keep
    return p, pd, m, cond


@pytest.mark.parametrize("drop", ["none", "mask_p0.2", "mask_p0", "nomask_p0.2"])
@pytest.mark.parametrize("L", P.SOFTMAX_LS)
def test_attn_softmax_forward_and_backward(L, drop):
    """fs2_attn_softmax / fs2_attn_softmax_backward with lens 0, 1, L - 1, L and L + 5, scores up to +-80.  Forward: NaN
    at every masked score changes nothing, p and pd are exactly 0 there; p is gated relative to p (1 + |s - max|), the
    condition number of exp.  Backward: large finite garbage in dpd at masked positions changes no bit of ds."""
    heads = 2
    lens = torch.tensor(P.SOFTMAX_LENS(L), device=DEV)
    B = lens.numel()
    p_drop = 0.2 if drop in ("mask_p0.2", "nomask_p0.2") else 0.0
    s = (rnd((B, heads, L, L), L) * 30).clamp(-80, 80)
    dmask = None
    if drop.startswith("mask"):
        dmask = (torch.rand((B, heads, L, L), generator=torch.Generator(device=DEV).manual_seed(L), device=DEV) >= 0.2).to(torch.uint8)
    keep = float(np.float32(1.0) / (np.float32(1.0) - np.float32(p_drop)))
    p_ref, pd_ref, m, cond = _softmax_ref(s, lens, keep, dmask, heads)
    s_nan = s.masked_fill(~m, NAN)
    n = B * heads * L * L
    p, pd = Guarded(n), Guarded(n)
    call("fs2_attn_softmax", s_nan.data_ptr(), lens.data_ptr(), None if dmask is None else dmask.data_ptr(), p_drop, B, heads, L, p.ptr, pd.ptr)
    p2, pd2 = torch.empty(n, device=DEV), torch.empty(n, device=DEV)
    call("fs2_attn_softmax", s.data_ptr(), lens.data_ptr(), None if dmask is None else dmask.data_ptr(), p_drop, B, heads, L, p2.data_ptr(), pd2.data_ptr())
    torch.cuda.synchronize()
    assert p.intact() and pd.intact()
    assert torch.equal(bits(p.v), bits(p2)) and torch.equal(bits(pd.v), bits(pd2)), "a masked score was read"
    mm = m.expand(B, heads, L, L).reshape(-1)
    assert bool((p.v[~mm] == 0).all()) and bool((pd.v[~mm] == 0).all())
    ch = P.softmax(L)["chain"]
    tiny = 2.0 ** -126 * m            # fp32's underflow threshold, absolute: exp(-160) is a float64 number but an fp32 zero
    gate("softmax.p", ratio(p.v, p_ref, p_ref * cond + tiny), ch)
    gate("softmax.p", ratio(pd.v, pd_ref, pd_ref * cond + tiny), ch)

    dpd = rnd((B, heads, L, L), L + 1)
    dpd_garbage = dpd.masked_fill(~m, 1e30)
    ds, ds2 = Guarded(n), torch.empty(n, device=DEV)
    call("fs2_attn_softmax_backward", p.ptr, dpd_garbage.data_ptr(), None if dmask is None else dmask.data_ptr(), p_drop, B, heads, L, ds.ptr)
    call("fs2_attn_softmax_backward", p.ptr, dpd.data_ptr(), None if dmask is None else dmask.data_ptr(), p_drop, B, heads, L, ds2.data_ptr())
    pv = p.v.double().reshape(B, heads, L, L)
    g = dpd.double() if dmask is None else dpd.double() * dmask.double() * keep
    want = pv * (g - (g * pv).sum(-1, keepdim=True))
    terms = pv * (g.abs() + (g * pv).abs().sum(-1, keepdim=True)) + tiny     # p (g - dot) can underflow
    torch.cuda.synchronize()
    assert ds.intact()
    assert torch.equal(ds.v, ds2), "garbage in dpd at a masked position reached ds"
    gate("softmax.ds", ratio(ds.v, want, terms), ch)
    free()


# ---- AttentionFn at bench scale ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,L", [(256, 100), (384, 800)])
def test_attention_fn_at_bench_scale(C, L):
    """B = 64, 2 heads, ragged lens including 1 and L, dropout 0.2.  Against float64 (terms: the same products on absolute
    values, ds's terms carried into dq, dk; the ceiling adds the score chain and exp's condition number); garbage
    (1e6 scale) in the q, k, v and dO rows past each length changes no bit of the valid context rows or of dq, dk, dv,
    and the gradient rows past each length are exactly 0."""
    B, heads = 64, 2
    dk = C // heads
    g = torch.Generator().manual_seed(L)
    lens = torch.randint(1, L + 1, (B,), generator=g)
    lens[0], lens[1] = L, 1
    lens = lens.to(DEV)
    q, k, v, dO = (rnd((B, L, C), L + i) for i in range(4))
    dmask = (torch.rand((B, heads, L, L), generator=torch.Generator(device=DEV).manual_seed(L + 9), device=DEV) >= 0.2).to(torch.uint8)
    pad = (torch.arange(L, device=DEV)[None] >= lens[:, None])[..., None]          # [B, L, 1]

    def run(qq, kk, vv, gg):
        leaves = [t.clone().requires_grad_() for t in (qq, kk, vv)]
        out = T.AttentionFn.apply(*leaves, lens, heads, 0.2, dmask)
        out.backward(gg)
        return out.detach(), [t.grad for t in leaves]

    out, grads = run(q, k, v, dO)
    junk = [torch.where(pad, rnd((B, L, C), 100 + i, 1e6), t) for i, t in enumerate((q, k, v, dO))]
    out_j, grads_j = run(*junk)
    valid = ~pad.expand(B, L, C)
    assert torch.equal(out[valid], out_j[valid]), "garbage past a length reached a valid context row"
    for a, b in zip(grads, grads_j):
        assert torch.equal(a, b), "garbage past a length reached a gradient"
        assert bool((a[~valid] == 0).all()), "a gradient row past the length is not 0"

    keep = float(np.float32(1.0) / np.float32(0.8))
    split = lambda t: t.double().view(B, L, heads, dk).transpose(1, 2)
    sc = 1.0 / math.sqrt(dk)
    Q, K_, V, G = (split(t) for t in (q, k, v, dO))
    s64 = Q @ K_.transpose(-1, -2) * sc
    p, pd, m, cond = _softmax_ref(s64, lens, keep, dmask, heads)
    del s64
    merge = lambda t: t.transpose(1, 2).reshape(B, L, C)
    chain = (dk + L + P.softmax(L)["chain"] + 2) * float(cond.max())
    del cond
    gate("attention", ratio(out, merge(pd @ V), merge(pd @ V.abs())), chain)
    gate("attention", ratio(grads[2], merge(pd.transpose(-1, -2) @ G), merge(pd.transpose(-1, -2) @ G.abs())), chain)
    gd = (G @ V.transpose(-1, -2)) * dmask.double() * keep
    ds = p * (gd - (gd * p).sum(-1, keepdim=True))
    t_ds = p * ((G.abs() @ V.abs().transpose(-1, -2)) * dmask.double() * keep + (gd * p).abs().sum(-1, keepdim=True))
    del gd, pd
    gate("attention", ratio(grads[0], merge(ds @ K_) * sc, merge(t_ds @ K_.abs()) * sc), chain)
    gate("attention", ratio(grads[1], merge(ds.transpose(-1, -2) @ Q) * sc, merge(t_ds.transpose(-1, -2) @ Q.abs()) * sc), chain)
    del p, ds, t_ds
    free()


# ---- embedding and positional encoding --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ids", ["mixed", "one_id"])
def test_embed_backward_and_embed_fn(ids):
    """fs2_embed_backward: dtable[id] += dy (row 0, the padding index, keeps its starting value exactly), dalpha +=
    sum dy . pe, a cancelling sum gated relative to sum |dy pe|; 'one_id': every row the same id (atomic contention).
    EmbedFn / fs2_embed_posenc forward: the fp32 expression table[id] + (alpha * pe) bit for bit."""
    B, Tn, C, n_sym = P.C2_B, P.C2_T, 256, 68
    g = torch.Generator().manual_seed(5)
    xs = torch.randint(0, n_sym, (B, Tn), generator=g)
    xs[:, -7:] = 0
    xs[0, 0] = n_sym - 1
    if ids == "one_id":
        xs.fill_(5)
    xs = xs.to(DEV)
    dy = rnd((B, Tn, C), 6)
    pe = rnd((Tn, C), 7)
    init = rnd((n_sym, C), 8)
    a0 = rnd(1, 9)
    dt, da = Guarded(n_sym * C, fill=init), Guarded(1, fill=a0)
    call("fs2_embed_backward", xs.data_ptr(), dy.data_ptr(), pe.data_ptr(), B, Tn, C, n_sym, dt.ptr, da.ptr)
    dy64 = dy.double().reshape(-1, C)
    flat = xs.reshape(-1)
    sel = flat > 0
    want = init.double().index_add(0, flat[sel], dy64[sel])
    terms = init.double().abs().index_add(0, flat[sel], dy64[sel].abs())
    prod = dy.double() * pe.double()[None]
    torch.cuda.synchronize()
    assert dt.intact() and da.intact()
    assert torch.equal(dt.v.reshape(n_sym, C)[0], init[0]), "the padding row's gradient changed"
    gate("embed.dtable", ratio(dt.v, want, terms), int(torch.bincount(flat, minlength=n_sym)[1:].max()) + 1)
    gate("embed.dalpha", ratio(da.v, a0.double() + prod.sum(), a0.double().abs() + prod.abs().sum()), P.embed_chain(B * Tn, C))
    # EmbedFn / PosEncFn
    table = rnd((n_sym, C), 10).requires_grad_()
    alpha = torch.tensor(1.3, device=DEV).requires_grad_()           # a 0-d parameter, as ScaledPositionalEncoding's
    out = T.EmbedFn.apply(xs, table, alpha, pe)
    want_out = table.detach()[xs] + alpha.detach() * pe[None]        # x + (alpha * pe): two roundings, as the kernel
    assert torch.equal(bits(out), bits(want_out))
    out.backward(dy)
    assert bool((table.grad[0] == 0).all())
    gate("embed.dtable", ratio(table.grad, want - init.double(), terms - init.double().abs()),
         int(torch.bincount(flat, minlength=n_sym)[1:].max()) + 1)
    gate("embed.dalpha", ratio(alpha.grad, prod.sum(), prod.abs().sum()), P.embed_chain(B * Tn, C))
    direct = torch.empty_like(out)
    call("fs2_embed_posenc", xs.data_ptr(), table.detach().data_ptr(), n_sym, pe.data_ptr(), alpha.detach().data_ptr(), B, Tn, C, direct.data_ptr())
    assert torch.equal(direct, out.detach())


def test_posenc_add_bit_for_bit_and_posenc_fn():
    """fs2_posenc_add: x + (alpha * pe[t]) with two roundings, bit for bit, at the decoder's c2 shape; PosEncFn's dalpha
    through fs2_embed_backward with no table."""
    B, Lf, C = P.C2_B, P.C2_L, 384
    x = rnd((B, Lf, C), 1)
    pe = rnd((Lf, C), 2)
    alpha = torch.tensor(0.77, device=DEV)
    y = Guarded(B * Lf * C)
    call("fs2_posenc_add", x.data_ptr(), pe.data_ptr(), alpha.data_ptr(), B, Lf, C, y.ptr)
    want = x + alpha * pe[None]
    torch.cuda.synchronize()
    assert y.intact() and torch.equal(bits(y.v), bits(want).reshape(-1))
    ar = alpha.clone().requires_grad_()
    xr = x.clone().requires_grad_()
    out = T.PosEncFn.apply(xr, ar, pe)
    assert torch.equal(bits(out), bits(want))
    dy = rnd((B, Lf, C), 3)
    out.backward(dy)
    assert torch.equal(xr.grad, dy)
    prod = dy.double() * pe.double()[None]
    da = Guarded(1, fill=torch.tensor([0.25], device=DEV))
    call("fs2_embed_backward", None, dy.data_ptr(), pe.data_ptr(), B, Lf, C, 0, None, da.ptr)
    torch.cuda.synchronize()
    assert da.intact()
    gate("embed.dalpha", ratio(da.v, 0.25 + prod.sum(), 0.25 + prod.abs().sum()), P.embed_chain(B * Lf, C))
    gate("embed.dalpha", ratio(ar.grad, prod.sum(), prod.abs().sum()), P.embed_chain(B * Lf, C))
    free()


# ---- one-hot Linear (pitch / energy embedding) ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("ids", ["spread", "one_id"])
def test_onehot_linear(ids):
    """fs2_onehot_linear_forward bit for bit (x + (W[:, id] + b)); fs2_onehot_linear_backward dW[:, id] += dy and
    db += sum dy from seeded values; ids 0 and n_bins - 1, or every row one id; OneHotLinearAddFn the same."""
    B, Lf, C, nb = P.C2_B, P.C2_L, 256, 256
    rows = B * Lf
    g = torch.Generator().manual_seed(3)
    idv = torch.randint(0, nb, (rows,), generator=g)
    idv[:5] = 0
    idv[5:10] = nb - 1
    if ids == "one_id":
        idv.fill_(nb - 1)
    idv = idv.to(DEV)
    x = rnd((rows, C), 4)
    W, b = rnd((C, nb), 5), rnd(C, 6)
    y = Guarded(rows * C)
    call("fs2_onehot_linear_forward", x.data_ptr(), idv.data_ptr(), W.data_ptr(), b.data_ptr(), rows, C, nb, y.ptr)
    want = x + (W[:, idv].T + b)
    torch.cuda.synchronize()
    assert y.intact() and torch.equal(bits(y.v), bits(want).reshape(-1))
    dy = rnd((rows, C), 7)
    iW, ib = rnd((C, nb), 8), rnd(C, 9)
    dW, db = Guarded(C * nb, fill=iW), Guarded(C, fill=ib)
    call("fs2_onehot_linear_backward", idv.data_ptr(), dy.data_ptr(), rows, C, nb, dW.ptr, db.ptr)
    dy64 = dy.double()
    want_W = iW.double().T.index_add(0, idv, dy64).T
    terms_W = iW.double().abs().T.index_add(0, idv, dy64.abs()).T
    torch.cuda.synchronize()
    assert dW.intact() and db.intact()
    chain = int(torch.bincount(idv, minlength=nb).max()) + 1
    gate("onehot.dW", ratio(dW.v, want_W, terms_W), chain)
    gate("colsum", ratio(db.v, ib.double() + dy64.sum(0), ib.double().abs() + dy64.abs().sum(0)), P.colsum(rows, C)["chain"])
    xr, Wr, br = x.clone().requires_grad_(), W.clone().requires_grad_(), b.clone().requires_grad_()
    out = T.OneHotLinearAddFn.apply(xr, idv, Wr, br)
    assert torch.equal(bits(out), bits(want))
    out.backward(dy)
    assert torch.equal(xr.grad, dy)
    gate("onehot.dW", ratio(Wr.grad, want_W - iW.double(), terms_W - iW.double().abs()), chain)
    free()


# ---- LengthRegulator backward ------------------------------------------------------------------------------------------------------
def _lr_reference(dout, d, ilens, Lcap):
    """float64 dhs[b, i] = sum of dout[b, j] over the frames j < Lcap copied from phoneme i < ilens[b]; and the terms."""
    B, Tn = d.shape
    C = dout.shape[-1]
    want = torch.zeros(B, Tn, C, dtype=torch.float64, device=DEV)
    terms = torch.zeros_like(want)
    for b in range(B):
        il = min(int(ilens[b]), Tn)
        reps = d[b, :il].clamp_min(0).to(torch.int64)
        owner = torch.repeat_interleave(torch.arange(il, device=DEV), reps.to(DEV))[:Lcap]
        n = owner.numel()
        src = dout[b, :n].double()
        want[b].index_add_(0, owner, src)
        terms[b].index_add_(0, owner, src.abs())
    return want, terms


def _lr_case(kind):
    if kind == "edges":
        Tn, Lcap, C = 12, 600, 200
        d = torch.tensor([[0, 3, 0, 500, 2, 0, 4, 0, 9, 9, 9, 9],          # leading / interior / trailing zeros, ilens < T, a 500-frame phoneme
                          [5] * 12,                                      # ilens = 0
                          [100] * 12,                                    # sum 1200 > Lcap: clipped
                          [1, 1, 1, 1, 1, 7, 7, 7, 7, 7, 7, 7],          # durations past ilens ignored
                          [0, 0, 300, 0, 0, 0, 150, 150, 0, 0, 0, 0]])   # sum exactly Lcap, trailing zeros
        ilens = torch.tensor([8, 0, 12, 5, 12])
    else:                                                               # c2: 64 x 100 phonemes, 800 frames
        Tn, Lcap, C = P.C2_T, P.C2_L, 256
        g = torch.Generator().manual_seed(11)
        ilens = torch.randint(40, Tn + 1, (P.C2_B,), generator=g)
        ilens[0] = Tn
        d = torch.randint(0, 15, (P.C2_B, Tn), generator=g)
        d[:, ::9] = 0
    return d, ilens, Tn, Lcap, C


@pytest.mark.parametrize("kind", ["edges", "c2"])
def test_length_regulator_backward(kind):
    """fs2_length_regulator_backward on a cum the caller built: NaN in dout frames past an utterance's duration sum and
    garbage in cum past ilens change nothing; rows past ilens are exactly 0."""
    d, ilens, Tn, Lcap, C = _lr_case(kind)
    B = d.shape[0]
    cum = torch.cumsum(d, 1)
    cum = torch.where(torch.arange(Tn)[None] < ilens[:, None], cum, torch.full_like(cum, 0x7FFF0000)).to(torch.int32)
    used = torch.tensor([min(int(cum[b, int(ilens[b]) - 1]) if ilens[b] > 0 else 0, Lcap) for b in range(B)])
    dout = rnd((B, Lcap, C), Tn)
    dout = dout.masked_fill((torch.arange(Lcap)[None] >= used[:, None]).to(DEV)[..., None], NAN)
    dhs = Guarded(B * Tn * C)
    il = ilens.to(DEV)
    call("fs2_length_regulator_backward", dout.data_ptr(), cum.to(DEV).data_ptr(), il.data_ptr(), B, Tn, C, Lcap, dhs.ptr)
    want, terms = _lr_reference(torch.nan_to_num(dout, nan=0.0), d, ilens, Lcap)
    torch.cuda.synchronize()
    assert dhs.intact()
    got = dhs.v.reshape(B, Tn, C)
    past = (torch.arange(Tn)[None] >= ilens[:, None]).to(DEV)
    assert bool((got[past] == 0).all()), "a row past ilens is not 0"
    gate("length_regulator", ratio(got, want, terms), int(d.max()) + 1)


@pytest.mark.parametrize("dtype", [torch.int64, torch.int32, torch.float32], ids=str)
def test_length_regulator_fn(dtype):
    """LengthRegulatorFn with durations as int64, int32 and float32: forward is the expansion, backward the per-phoneme sum;
    NaN in the incoming gradient past each utterance's frames changes nothing."""
    B, Tn, C = 4, 15, 256
    g = torch.Generator().manual_seed(2)
    d = torch.randint(0, 6, (B, Tn), generator=g)
    d[0, :3] = 0
    d[1, -4:] = 0
    d[2, 7] = 40
    ilens = torch.tensor([Tn, 11, 9, 13])
    tot = torch.stack([d[b, :ilens[b]].sum() for b in range(B)])
    L = int(tot.max())
    hs = rnd((B, Tn, C), 3).requires_grad_()
    out = T.LengthRegulatorFn.apply(hs, d.to(dtype).to(DEV), ilens.to(DEV), L)
    dy = rnd((B, L, C), 4).masked_fill((torch.arange(L)[None] >= tot[:, None]).to(DEV)[..., None], NAN)
    out.backward(dy)
    want, terms = _lr_reference(torch.nan_to_num(dy, nan=0.0), d, ilens, L)
    assert torch.isfinite(hs.grad).all()
    gate("length_regulator", ratio(hs.grad, want, terms), int(d.max()) + 1)
    for b in range(B):
        il = int(ilens[b])
        rows = torch.repeat_interleave(hs.detach()[b, :il], d[b, :il].to(DEV), dim=0)
        assert torch.equal(out[b, :rows.shape[0]], rows) and bool((out[b, rows.shape[0]:] == 0).all())
        assert bool((hs.grad[b, il:] == 0).all())


# ---- predictor head ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [256, 384])
@pytest.mark.parametrize("BL", [(5, 845), (P.C2_B, P.C2_L)], ids=lambda bl: "rows%d" % (bl[0] * bl[1]))
def test_rowdot_forward_and_backward(BL, C):
    """fs2_rowdot: y = x . w + bias, exactly 0 at padded rows; fs2_rowdot_backward: NaN in dy at padded rows must not
    reach dx, dw or dbias; dw, dbias from seeded values; RowDotFn the same."""
    B, L = BL
    rows = B * L
    g = torch.Generator().manual_seed(rows + C)
    lens = torch.randint(1, L + 1, (B,), generator=g)
    lens[0] = L
    lens = lens.to(DEV)
    x = rnd((rows, C), rows + C)
    w, bias = rnd(C, 1), rnd(1, 2)
    pad = (torch.arange(L, device=DEV)[None] >= lens[:, None]).reshape(-1)
    y = Guarded(rows)
    call("fs2_rowdot", x.data_ptr(), w.data_ptr(), bias.data_ptr(), lens.data_ptr(), rows, L, C, y.ptr)
    x64 = x.double()
    want = x64 @ w.double() + bias.double()
    terms = x64.abs() @ w.double().abs() + bias.double().abs()
    torch.cuda.synchronize()
    assert y.intact() and bool((y.v[pad] == 0).all())
    ch = P.rowdot_chain(rows, C)
    gate("rowdot.y", ratio(y.v[~pad], want[~pad], terms[~pad]), ch["y"])

    dy = rnd(rows, 3).masked_fill(pad, NAN)
    iw, ib = rnd(C, 4), rnd(1, 5)
    dx, dw, db = Guarded(rows * C), Guarded(C, fill=iw), Guarded(1, fill=ib)
    call("fs2_rowdot_backward", x.data_ptr(), w.data_ptr(), dy.data_ptr(), lens.data_ptr(), rows, L, C, dx.ptr, dw.ptr, db.ptr)
    g64 = torch.nan_to_num(dy, nan=0.0).double()
    torch.cuda.synchronize()
    assert dx.intact() and dw.intact() and db.intact()
    assert torch.equal(bits(dx.v.reshape(rows, C)), bits((g64[:, None] * w.double()[None]).float())), "dx = g * w, one rounding"
    gate("rowdot.dw", ratio(dw.v, iw.double() + g64 @ x64, iw.double().abs() + g64.abs() @ x64.abs()), ch["dw"])
    gate("rowdot.dbias", ratio(db.v, ib.double() + g64.sum(), ib.double().abs() + g64.abs().sum()), ch["dbias"])

    xr, wr, br = x.reshape(B, L, C).clone().requires_grad_(), w.reshape(1, C).clone().requires_grad_(), bias.clone().requires_grad_()
    yf = T.RowDotFn.apply(xr, wr, br, lens)
    assert torch.equal(yf.reshape(-1), y.v)
    yf.backward(dy.reshape(B, L))
    assert torch.isfinite(xr.grad).all() and torch.isfinite(wr.grad).all() and torch.isfinite(br.grad).all()
    gate("rowdot.dw", ratio(wr.grad.reshape(-1), g64 @ x64, g64.abs() @ x64.abs()), ch["dw"])
    gate("rowdot.dbias", ratio(br.grad, g64.sum(), g64.abs().sum()), ch["dbias"])
    free()


# ---- losses ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ds_dtype", [torch.int64, torch.int32, torch.float32], ids=str)
def test_masked_losses_and_loss_backward(ds_dtype):
    """fs2_masked_losses / fs2_loss_backward / LossFn (fastspeech.py:277-324 with use_masking) against float64: ys passed
    unsliced (ld_ys_time > L); NaN (garbage for integer durations) at every padded position of every input changes no
    value, and the gradients are exactly 0 there; L1 at zero difference has gradient 0 (torch's sign); grad_loss != 1."""
    B, Tn, L, odim = 4, 20, 150, 80
    ilens = torch.tensor([20, 13, 1, 7], device=DEV)
    olens = torch.tensor([150, 96, 3, 60], device=DEV)
    Ly = L + 17
    tvalid = torch.arange(Tn, device=DEV)[None] < ilens[:, None]
    lvalid = torch.arange(L, device=DEV)[None] < olens[:, None]
    before, after = rnd((B, L, odim), 1), rnd((B, L, odim), 2)
    ys = rnd((B, Ly, odim), 3)
    ys[:, :L][:, ::5] = before[:, ::5]                         # zero differences
    d_out, e_out, p_out, es, ps = rnd((B, Tn), 4), rnd((B, L), 5), rnd((B, L), 6), rnd((B, L), 7), rnd((B, L), 8)
    g = torch.Generator().manual_seed(9)
    ds = torch.randint(0, 12, (B, Tn), generator=g).to(DEV)
    ds64 = ds.double()
    # poison every padded position
    lv3 = lvalid[..., None]
    before_n, after_n = before.masked_fill(~lv3, NAN), after.masked_fill(~lv3, NAN)
    ys_n = ys.clone()
    ys_n[:, :L] = ys[:, :L].masked_fill(~lv3, NAN)
    ys_n[:, L:] = NAN
    d_n = d_out.masked_fill(~tvalid, NAN)
    e_n, p_n, es_n, ps_n = (t.masked_fill(~lvalid, NAN) for t in (e_out, p_out, es, ps))
    ds_n = ds.to(ds_dtype).masked_fill(~tvalid, NAN if ds_dtype == torch.float32 else -12345)

    ni, no = float(ilens.sum()), float(olens.sum())
    yv = ys[:, :L].double()
    l_b = ((before.double() - yv).abs() * lv3).sum() / (no * odim)
    l_a = ((after.double() - yv).abs() * lv3).sum() / (no * odim)
    dd = (d_out.double() - torch.log(ds64 + 1)) * tvalid
    l_d = (dd ** 2).sum() / ni
    de, dp = (e_out.double() - es.double()) * lvalid, (p_out.double() - ps.double()) * lvalid
    l_e, l_p = (de ** 2).sum() / no, (dp ** 2).sum() / no
    want7 = torch.stack([l_b + l_a, l_b, l_a, l_d, l_e, l_p, l_b + l_a + l_d + l_e + l_p])
    out7 = torch.empty(7, device=DEV)
    scratch = torch.empty(16, dtype=torch.float64, device=DEV)
    call("fs2_masked_losses", before_n.data_ptr(), after_n.data_ptr(), ys_n.data_ptr(), Ly, d_n.data_ptr(), ds_n.data_ptr(), _lib.dur_dtype(ds_n),
         e_n.data_ptr(), p_n.data_ptr(), es_n.data_ptr(), ps_n.data_ptr(), ilens.data_ptr(), olens.data_ptr(), B, Tn, L, odim, out7.data_ptr(),
         scratch.data_ptr())
    n_terms = int(olens.sum()) * odim
    gate("loss.values", ratio(out7, want7, want7), n_terms)

    gl = torch.tensor([0.7], device=DEV)
    outs = [Guarded(B * L * odim), Guarded(B * L * odim), Guarded(B * Tn), Guarded(B * L), Guarded(B * L)]
    call("fs2_loss_backward", before_n.data_ptr(), after_n.data_ptr(), ys_n.data_ptr(), Ly, d_n.data_ptr(), ds_n.data_ptr(), _lib.dur_dtype(ds_n),
         e_n.data_ptr(), p_n.data_ptr(), es_n.data_ptr(), ps_n.data_ptr(), ilens.data_ptr(), olens.data_ptr(), B, Tn, L, odim, gl.data_ptr(),
         *[o.ptr for o in outs])
    g7 = float(np.float32(0.7))
    cm = g7 / (no * odim)
    w_b = cm * torch.sign(before.double() - yv) * lv3
    w_a = cm * torch.sign(after.double() - yv) * lv3
    w_d = g7 * 2 * dd / ni
    t_d = g7 * 2 * (d_out.double().abs() + torch.log(ds64 + 1)) * tvalid / ni
    w_e, w_p = g7 * 2 * de / no, g7 * 2 * dp / no
    t_e = g7 * 2 * (e_out.double().abs() + es.double().abs()) * lvalid / no
    t_p = g7 * 2 * (p_out.double().abs() + ps.double().abs()) * lvalid / no
    torch.cuda.synchronize()
    assert all(o.intact() for o in outs)
    got = [o.v for o in outs]
    gate("loss.grads", ratio(got[0], w_b, w_b.abs()), 6)
    gate("loss.grads", ratio(got[1], w_a, w_a.abs()), 6)
    gate("loss.grads", ratio(got[2], w_d, t_d), 6)
    gate("loss.grads", ratio(got[3], w_e, t_e), 6)
    gate("loss.grads", ratio(got[4], w_p, t_p), 6)
    zero_diff = (before.double() == yv) & lv3
    assert bool(zero_diff.any()) and bool((got[0].reshape(B, L, odim)[zero_diff] == 0).all())
    assert bool((got[0].reshape(B, L, odim)[~lv3.expand(B, L, odim)] == 0).all())
    assert bool((got[2].reshape(B, Tn)[~tvalid] == 0).all()) and bool((got[3].reshape(B, L)[~lvalid] == 0).all())

    # LossFn: the same two entries behind autograd
    leaves = [t.clone().requires_grad_() for t in (before_n, after_n, d_n, e_n, p_n)]
    o7 = T.LossFn.apply(*leaves, ys_n, ds_n, es_n, ps_n, ilens, olens)
    assert torch.equal(o7, out7)
    (o7[6] * 0.7).backward()
    for leaf, o in zip(leaves, got):
        assert torch.equal(leaf.grad.reshape(-1), o)


# ---- coverage of the file by its own tests ----------------------------------------------------------------------------------------
def test_every_gate_is_used():
    src = open(__file__).read()
    tree = ast.parse(src)
    used = {n.args[0].value for n in ast.walk(tree) if isinstance(n, ast.Call) and getattr(n.func, "id", None) == "gate"
            and isinstance(n.args[0], ast.Constant)}
    assert used == set(GATES), set(GATES) ^ used
