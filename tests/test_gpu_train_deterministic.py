"""The deterministic train mode on the H100 (DESIGN.md §26).

* every `_det` entry against float64 at tests/_train_plan.py's cases, gated by its a-priori chain bound from
  tests/_det_plan.py (`max|err| / sum|terms| <= n_chain * 2^-24`), with sentinel guard bands and nonzero starting values;
* every `_det` entry bit-identical over three calls with the workspace pre-filled with NaN, zeros and random bits, the
  inputs copied to another allocation for the last call; the scatter entries at one id, all ids distinct, padding id 0,
  ids >= n, and rows = 0, 1 and 51,200;
* three full train steps (forward, backward, NoamAdam.clip_and_step) on a ragged batch in fp32, tf32 and tf32 + flash,
  single- and multi-speaker, twice from the same weights and seed: every loss, report value, gradient, parameter, Adam
  state and BatchNorm running statistic equal; the same run in a subprocess gives the same SHA-256;
* one deterministic step against one default step within tests/test_gpu_train.py's gates;
* torch.use_deterministic_algorithms(True) on a model built without the flag: the same bits, no error;
* two deterministic aligner trainings: identical weights and durations;
* the kernels torch.profiler records in deterministic steps: none of them holds a floating-point atomic.
Needs an H100: run with `-m gpu`."""
import hashlib
import io
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _det_plan as D
import _train_plan as P
from fastspeech2_b200 import FeedForwardTransformer, _lib, synthetic_state_dict
from fastspeech2_b200 import optim as O
from fastspeech2_b200 import train as T
from fastspeech2_b200._kernel_module import query_bytes
from fastspeech2_b200.hparams import load_hp
from fastspeech2_b200.synthetic import make_batch

pytestmark = pytest.mark.gpu
KEYS = ("xs", "ilens", "ys", "olens", "ds", "es", "ps")
HERE = os.path.dirname(os.path.abspath(__file__))
FILLS = ("nan", "zeros", "random")
GUARD = 64                         # sentinel floats after every output


def lib():
    return _lib.load()


def st():
    return _lib.stream_ptr(torch.device("cuda"))


def workspace(entry, fill, *shape):
    n = query_bytes(entry + "_ws_bytes", *shape)
    ws = torch.empty((max(n, 16) // 4 + 4,), dtype=torch.float32, device="cuda")
    if fill == "nan":
        ws.fill_(float("nan"))
    elif fill == "zeros":
        ws.zero_()
    else:
        ws.view(torch.int32).copy_(torch.randint(-2**31, 2**31 - 1, ws.shape, dtype=torch.int32, device="cuda"))
    return ws, n


def guarded(t):
    """t (flattened) followed by GUARD sentinels, as a fresh buffer; returns (buffer, view of t's part)"""
    buf = torch.full((t.numel() + GUARD,), 12345.0, dtype=torch.float32, device="cuda")
    buf[: t.numel()] = t.reshape(-1).to(device="cuda", dtype=torch.float32)
    return buf, buf[: t.numel()].view(t.shape)


def check_guard(buf, n):
    assert bool((buf[n:] == 12345.0).all()), "wrote past the output"


def gate(got, want, terms, chain, what):
    err = float((got.double().cpu() - want).abs().max())
    bound = chain * D.U24 * float(terms.max()) + 1e-30
    assert err <= bound, f"{what}: max err {err:.3e} > {chain} * 2^-24 * sum|terms| = {bound:.3e}"


def three_calls(run):
    """run(fill, copy_inputs) -> tuple of output tensors; the three calls must agree bit for bit."""
    outs = [run(fill, i == 2) for i, fill in enumerate(FILLS)]
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a, b.view(torch.int32) if b.dtype == torch.float32 else b)
    return outs[0]


def fresh(t, copy):
    """t, or a copy of it in another allocation.  Callers keep the copy in a local until the call is synchronised: a
    temporary would be freed before the kernel runs and its block handed to the next allocation."""
    return t.clone() if copy else t


def nonempty(t):
    """t on the device, or a one-element stand-in when t is empty (an empty tensor's pointer is NULL, which the entries refuse)"""
    return t.cuda() if t.numel() else torch.zeros(1, dtype=t.dtype, device="cuda")


# ---- colsum ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", P.COLSUM_ROWS)
@pytest.mark.parametrize("C", [1, 33, 256])
def test_colsum_det(rows, C):
    g = torch.Generator().manual_seed(rows * 7 + C)
    x = torch.randn(rows, C, generator=g)
    out0 = torch.randn(C, generator=g)
    xc = x.cuda()

    def run(fill, copy):
        buf, out = guarded(out0)
        ws, n = workspace("fs2_colsum_det", fill, rows, C)
        xi = fresh(xc, copy)
        _lib.check(lib().fs2_colsum_det(xi.data_ptr(), rows, C, out.data_ptr(), ws.data_ptr(), n, st()), "fs2_colsum_det")
        torch.cuda.synchronize()
        check_guard(buf, C)
        return (out.clone(),)

    (got,) = three_calls(run)
    want = out0.double() + x.double().sum(0)
    gate(got, want, out0.double().abs() + x.double().abs().sum(0), D.colsum_chain(rows), f"colsum rows={rows} C={C}")


# ---- fp32 weight gradient -----------------------------------------------------------------------------------------------------
WGRAD_CASES = [(3, 70, 256, 256, 1), (3, 70, 1024, 256, 9), (64, 100, 256, 256, 1), (3, 100, 80, 256, 5), (64, 800, 80, 384, 1),
               (3, 2, 80, 256, 5)] + P.WGRAD_TAIL_CASES


@pytest.mark.parametrize("case", WGRAD_CASES)
def test_conv_wgrad_det(case):
    B, L, N, K, taps = case
    g = torch.Generator().manual_seed(sum(case))
    dy, x = torch.randn(B, L, N, generator=g), torch.randn(B, L, K, generator=g)
    dw0, db0 = torch.randn(N, K, taps, generator=g), torch.randn(N, generator=g)
    dyc, xc = dy.cuda(), x.cuda()

    def run(fill, copy):
        bw, dw = guarded(dw0)
        bb, db = guarded(db0)
        ws, n = workspace("fs2_conv_wgrad_det", fill, B, L, N, K, taps)
        a, b = fresh(dyc, copy), fresh(xc, copy)
        _lib.check(lib().fs2_conv_wgrad_det(a.data_ptr(), b.data_ptr(), B, L, N, K, taps, dw.data_ptr(), db.data_ptr(), ws.data_ptr(), n, st()),
                   "fs2_conv_wgrad_det")
        torch.cuda.synchronize()
        check_guard(bw, dw0.numel()); check_guard(bb, N)
        return dw.clone(), db.clone()

    gw, gb = three_calls(run)
    pad = (taps - 1) // 2
    xp = torch.nn.functional.pad(x.double(), (0, 0, pad, pad))
    want = dw0.double().clone()
    terms = dw0.double().abs().clone()
    for j in range(taps):
        xs = xp[:, j: j + L]
        want[:, :, j] += torch.einsum("bln,blk->nk", dy.double(), xs)
        terms[:, :, j] += torch.einsum("bln,blk->nk", dy.double().abs(), xs.abs())
    gate(gw, want, terms, D.wgrad_chain(*case), f"wgrad {case}")
    gate(gb, db0.double() + dy.double().sum((0, 1)), db0.double().abs() + dy.double().abs().sum((0, 1)), D.colsum_chain(B * L), f"dbias {case}")


# ---- LayerNorm backward ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", P.LN_ROWS)
@pytest.mark.parametrize("C", P.LN_CS)
def test_layernorm_backward_det(rows, C):
    g = torch.Generator().manual_seed(rows + C)
    x = torch.randn(rows, C, generator=g) * 2 + 0.3
    dy = torch.randn(rows, C, generator=g)
    gamma = 1 + 0.2 * torch.randn(C, generator=g)
    dg0, db0 = torch.randn(C, generator=g), torch.randn(C, generator=g)
    xc, dyc, gc = x.cuda(), dy.cuda(), gamma.cuda()

    def run(fill, copy):
        bg, dg = guarded(dg0)
        bb, db = guarded(db0)
        dx = torch.full((rows * C + GUARD,), float("nan"), device="cuda")
        dx[rows * C:] = 12345.0
        ws, n = workspace("fs2_layernorm_backward_det", fill, rows, C)
        a, b = fresh(xc, copy), fresh(dyc, copy)
        _lib.check(lib().fs2_layernorm_backward_det(a.data_ptr(), b.data_ptr(), gc.data_ptr(), 1e-5, rows, C, dx.data_ptr(), dg.data_ptr(),
                                                    db.data_ptr(), ws.data_ptr(), n, st()), "fs2_layernorm_backward_det")
        torch.cuda.synchronize()
        check_guard(bg, C); check_guard(bb, C); check_guard(dx, rows * C)
        return dg.clone(), db.clone(), dx[: rows * C].clone()

    dg, db, dx = three_calls(run)
    xd = x.double()
    xhat = (xd - xd.mean(1, keepdim=True)) / torch.sqrt(xd.var(1, unbiased=False, keepdim=True) + 1e-5)
    chain = D.layernorm_chain(rows)
    gate(dg, dg0.double() + (dy.double() * xhat).sum(0), dg0.double().abs() + (dy.double() * xhat).abs().sum(0), chain, "dgamma")
    gate(db, db0.double() + dy.double().sum(0), db0.double().abs() + dy.double().abs().sum(0), chain, "dbeta")
    # dx: the same per-row math as the default entry, bit for bit
    dx_def = torch.empty(rows * C, device="cuda")
    z = torch.zeros(C, device="cuda")
    _lib.check(lib().fs2_layernorm_backward(xc.data_ptr(), dyc.data_ptr(), gc.data_ptr(), 1e-5, rows, C, dx_def.data_ptr(), z.data_ptr(),
                                            z.clone().data_ptr(), st()), "fs2_layernorm_backward")
    assert torch.equal(dx, dx_def)


# ---- BatchNorm --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", P.BN_ROWS)
@pytest.mark.parametrize("C", P.BN_CS)
def test_batchnorm_det(rows, C):
    g = torch.Generator().manual_seed(rows * 3 + C)
    x = torch.randn(rows, C, generator=g) * 1.5 + 0.7
    dy = torch.randn(rows, C, generator=g)
    gamma, beta = 1 + 0.1 * torch.randn(C, generator=g), torch.randn(C, generator=g)
    rm0, rv0 = torch.randn(C, generator=g), torch.rand(C, generator=g) + 0.5
    dg0, db0 = torch.randn(C, generator=g), torch.randn(C, generator=g)
    xc, dyc, gc, bc = x.cuda(), dy.cuda(), gamma.cuda(), beta.cuda()

    def run(fill, copy):
        rm, rv = rm0.cuda(), rv0.cuda()
        stats, y = torch.empty(2 * C, device="cuda"), torch.empty(rows, C, device="cuda")
        ws, n = workspace("fs2_batchnorm_train_det", fill, rows, C)
        a, b = fresh(xc, copy), fresh(dyc, copy)
        _lib.check(lib().fs2_batchnorm_train_det(a.data_ptr(), rows, C, gc.data_ptr(), bc.data_ptr(), 1e-5, 0.1, 0, rm.data_ptr(), rv.data_ptr(),
                                                 stats.data_ptr(), y.data_ptr(), ws.data_ptr(), n, st()), "fs2_batchnorm_train_det")
        bg, dg = guarded(dg0)
        bb, db = guarded(db0)
        dx = torch.empty(rows, C, device="cuda")
        ws2, n2 = workspace("fs2_batchnorm_backward_det", fill, rows, C)
        _lib.check(lib().fs2_batchnorm_backward_det(a.data_ptr(), b.data_ptr(), stats.data_ptr(), gc.data_ptr(), 1e-5, rows, C,
                                                    dx.data_ptr(), dg.data_ptr(), db.data_ptr(), ws2.data_ptr(), n2, st()), "fs2_batchnorm_backward_det")
        torch.cuda.synchronize()
        check_guard(bg, C); check_guard(bb, C)
        return stats.clone(), y, rm, rv, dx, dg.clone(), db.clone()

    stats, y, rm, rv, dx, dg, db = three_calls(run)
    xd = x.double()
    mean, var = xd.mean(0), xd.var(0, unbiased=False)
    chain = P.bn(rows)["chain"]
    gate(stats[:C], mean, xd.abs().mean(0), chain, "mean")
    gate(stats[C:], var, (xd - mean).pow(2).mean(0) + mean.pow(2), chain, "var")
    xhat = (xd - mean) / torch.sqrt(var + 1e-5)
    gate(dg, dg0.double() + (dy.double() * xhat).sum(0), dg0.double().abs() + (dy.double() * xhat).abs().sum(0), chain, "dgamma")
    gate(db, db0.double() + dy.double().sum(0), db0.double().abs() + dy.double().abs().sum(0), chain, "dbeta")


# ---- scatter by id: embedding table and one-hot Linear ----------------------------------------------------------------------------
def scatter_ids(kind, rows, n, g):
    if kind == "one_id":
        return torch.full((rows,), max(n - 1, 1), dtype=torch.int64)
    if kind == "distinct":
        return torch.arange(rows, dtype=torch.int64) % n
    if kind == "padding":
        ids = torch.randint(0, n, (rows,), generator=g)
        ids[::3] = 0
        return ids
    if kind == "out_of_range":
        ids = torch.randint(0, n + 40, (rows,), generator=g)
        ids[::5] = -3
        return ids
    return torch.randint(0, n, (rows,), generator=g)


SCATTER_CASES = [("one_id", 51200), ("distinct", 256), ("padding", 4225), ("out_of_range", 4225), ("random", 0), ("random", 1),
                 ("random", 51200)]


@pytest.mark.parametrize("kind,rows", SCATTER_CASES)
def test_onehot_linear_backward_det(kind, rows):
    C, nb = 384, 256
    g = torch.Generator().manual_seed(rows + len(kind))
    ids = scatter_ids(kind, rows, nb, g)
    dy = torch.randn(rows, C, generator=g)
    dW0, db0 = torch.randn(C, nb, generator=g), torch.randn(C, generator=g)
    idc, dyc = nonempty(ids), nonempty(dy)

    def run(fill, copy):
        bw, dW = guarded(dW0)
        bb, db = guarded(db0)
        ws, n = workspace("fs2_onehot_linear_backward_det", fill, rows, C, nb)
        a, b = fresh(idc, copy), fresh(dyc, copy)
        _lib.check(lib().fs2_onehot_linear_backward_det(a.data_ptr(), b.data_ptr(), rows, C, nb, dW.data_ptr(),
                                                        db.data_ptr(), ws.data_ptr() if n else None, n, st()), "fs2_onehot_linear_backward_det")
        torch.cuda.synchronize()
        check_guard(bw, C * nb); check_guard(bb, C)
        return dW.clone(), db.clone()

    dW, db = three_calls(run)
    valid = (ids >= 0) & (ids < nb)
    want, terms = dW0.double().clone(), dW0.double().abs().clone()
    want.index_add_(1, ids[valid], dy.double()[valid].t())
    terms.index_add_(1, ids[valid], dy.double().abs()[valid].t())
    counts = torch.bincount(ids[valid], minlength=nb)
    gate(dW, want, terms, D.scatter_chain(int(counts.max()) if rows else 0), f"dW {kind} {rows}")
    untouched = counts == 0
    assert torch.equal(dW.cpu()[:, untouched], dW0[:, untouched])
    if rows:
        gate(db, db0.double() + dy.double().sum(0), db0.double().abs() + dy.double().abs().sum(0), D.colsum_chain(rows), "dbias")


@pytest.mark.parametrize("kind,rows", SCATTER_CASES)
def test_embed_backward_det(kind, rows):
    C, n_sym = 256, 68
    T_ = 50 if rows % 50 == 0 and rows else max(rows, 1)
    B = rows // T_ if rows else 0
    g = torch.Generator().manual_seed(rows * 5 + len(kind))
    ids = scatter_ids(kind, rows, n_sym, g)
    dy = torch.randn(rows, C, generator=g)
    pe = torch.randn(T_, C, generator=g)
    tab0, a0 = torch.randn(n_sym, C, generator=g), torch.randn(1, generator=g)
    idc, dyc, pec = nonempty(ids), nonempty(dy), pe.cuda()

    def run(fill, copy):
        bt, tab = guarded(tab0)
        ba, al = guarded(a0)
        ws, n = workspace("fs2_embed_backward_det", fill, B, T_, C, n_sym)
        a, b = fresh(idc, copy), fresh(dyc, copy)
        _lib.check(lib().fs2_embed_backward_det(a.data_ptr(), b.data_ptr(), pec.data_ptr(), B, T_, C, n_sym,
                                                tab.data_ptr(), al.data_ptr(), ws.data_ptr() if n else None, n, st()), "fs2_embed_backward_det")
        torch.cuda.synchronize()
        check_guard(bt, n_sym * C); check_guard(ba, 1)
        return tab.clone(), al.clone()

    tab, al = three_calls(run)
    valid = (ids > 0) & (ids < n_sym)
    want, terms = tab0.double().clone(), tab0.double().abs().clone()
    want.index_add_(0, ids[valid], dy.double()[valid])
    terms.index_add_(0, ids[valid], dy.double().abs()[valid])
    counts = torch.bincount(ids[valid], minlength=n_sym)
    gate(tab, want, terms, D.scatter_chain(int(counts.max()) if rows else 0), f"dtable {kind} {rows}")
    assert torch.equal(tab.cpu()[0], tab0[0]) and torch.equal(tab.cpu()[counts == 0], tab0[counts == 0])
    if rows:
        per = dy.double() * pe.double().repeat(B, 1)
        gate(al, a0.double() + per.sum(), a0.double().abs() + per.abs().sum(), D.dalpha_chain(rows, C), "dalpha")


# ---- rowdot backward --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", P.ROWDOT_ROWS + [1, 7])
def test_rowdot_backward_det(rows):
    C, L = 256, 25 if rows % 25 == 0 else rows
    g = torch.Generator().manual_seed(rows)
    x, w, dy = torch.randn(rows, C, generator=g), torch.randn(C, generator=g), torch.randn(rows, generator=g)
    lens = torch.randint(0, L + 1, (max(rows // L, 1),), generator=g)
    dw0, db0 = torch.randn(C, generator=g), torch.randn(1, generator=g)
    xc, wc, dyc, lc = x.cuda(), w.cuda(), dy.cuda(), lens.cuda()

    def run(fill, copy):
        bw, dw = guarded(dw0)
        bb, db = guarded(db0)
        dx = torch.empty(rows, C, device="cuda")
        ws, n = workspace("fs2_rowdot_backward_det", fill, rows, C)
        a, b = fresh(xc, copy), fresh(dyc, copy)
        _lib.check(lib().fs2_rowdot_backward_det(a.data_ptr(), wc.data_ptr(), b.data_ptr(), lc.data_ptr(), rows, L, C,
                                                 dx.data_ptr(), dw.data_ptr(), db.data_ptr(), ws.data_ptr(), n, st()), "fs2_rowdot_backward_det")
        torch.cuda.synchronize()
        check_guard(bw, C); check_guard(bb, 1)
        return dx, dw.clone(), db.clone()

    dx, dw, db = three_calls(run)
    t = torch.arange(rows) % L
    gm = torch.where(t < lens.repeat_interleave(L)[:rows], dy, torch.zeros(()))
    chain = D.rowdot_chain(rows)
    gate(dw, dw0.double() + (gm.double()[:, None] * x.double()).sum(0), dw0.double().abs() + (gm.double()[:, None] * x.double()).abs().sum(0),
         chain, "dw")
    gate(db, db0.double() + gm.double().sum(), db0.double().abs() + gm.double().abs().sum(), chain, "dbias")


# ---- masked losses ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,T_,L", [(2, 24, 190), (64, 100, 800), (3, 17, 400)])
def test_masked_losses_det(B, T_, L):
    bt = make_batch(B, T_, L, seed=B + L)
    g = torch.Generator().manual_seed(L)
    before, after = torch.randn(B, L, 80, generator=g).cuda(), torch.randn(B, L, 80, generator=g).cuda()
    d, e, p = torch.randn(B, T_, generator=g).cuda(), torch.randn(B, L, generator=g).cuda(), torch.randn(B, L, generator=g).cuda()
    ys, ds, es, ps = (bt[k].cuda().float().contiguous() if k != "ds" else bt[k].cuda() for k in ("ys", "ds", "es", "ps"))
    il, ol = bt["ilens"].cuda(), bt["olens"].cuda()

    def run(fill, copy):
        out7 = T.masked_losses(fresh(before, copy), fresh(after, copy), d, e, p, ys, ds, es, ps, il, ol, det=True)
        torch.cuda.synchronize()
        return (out7,)

    (got,) = three_calls(run)
    want = T.masked_losses(before, after, d, e, p, ys, ds, es, ps, il, ol, det=False)
    assert float((got - want).abs().max() / want.abs().max()) < 1e-6


# ---- full train steps -----------------------------------------------------------------------------------------------------------------
CONFIGS = [("fp32", "materialized"), ("tf32", "materialized"), ("tf32", "flash")]
SPEAKERS = torch.tensor([1, 3, 1, 0])


def make_model(prec, att, n_spk, det):
    hp = load_hp()
    hp["model"]["n_speakers"] = n_spk
    m = FeedForwardTransformer(68, 80, hp, train_precision=prec, train_attention=att, train_deterministic=det)
    sd = dict(synthetic_state_dict(0))
    if n_spk:
        sd["speaker_embed.weight"] = torch.randn(n_spk, m.dims.adim, generator=torch.Generator().manual_seed(9)) * 0.1
    m.load_state_dict(sd, strict=True)
    return m.cuda().train()


def three_steps(prec, att, n_spk, det, steps=3):
    """{name: tensor} after `steps` steps from synthetic weights on a ragged batch, plus every step's loss and report."""
    torch.manual_seed(0)
    m = make_model(prec, att, n_spk, det)
    opt = O.get_std_opt(m, 384, 100, 1.0)
    bt = {k: v.cuda() for k, v in make_batch(4, 40, 200, seed=5, ilens=[40, 31, 17, 25], olens=[200, 150, 90, 120]).items()}
    kw = {"speakers": SPEAKERS.cuda()} if n_spk else {}
    out = {}
    for s in range(steps):
        loss, rep = m(*[bt[k] for k in KEYS], **kw)
        loss.backward()
        out[f"loss{s}"] = loss.detach().clone()
        out[f"report{s}"] = torch.tensor([list(r.values())[0] for r in rep], dtype=torch.float64)
        for n, p in m.named_parameters():
            if p.grad is not None:
                out[f"grad{s}.{n}"] = p.grad.detach().clone()
        opt.clip_and_step(1.0)
        opt.zero_grad()
    for k, v in m.state_dict().items():
        out["state." + k] = v.detach().clone()
    for i, stt in opt.state_dict()["optimizer"]["state"].items():
        for k, v in stt.items():
            if torch.is_tensor(v):
                out[f"adam.{i}.{k}"] = v.detach().clone()
    return out


def digest(state):
    h = hashlib.sha256()
    for k in sorted(state):
        h.update(k.encode())
        h.update(state[k].detach().cpu().contiguous().numpy().tobytes())
    return h.hexdigest()


def assert_equal_states(a, b):
    assert a.keys() == b.keys()
    diff = [k for k in a if not torch.equal(a[k], b[k])]
    assert not diff, diff[:10]


@pytest.mark.parametrize("n_spk", [0, 4])
@pytest.mark.parametrize("prec,att", CONFIGS)
def test_three_steps_repeat_bit_for_bit(prec, att, n_spk):
    a = three_steps(prec, att, n_spk, det=True)
    b = three_steps(prec, att, n_spk, det=True)
    assert_equal_states(a, b)
    assert any(k.startswith("state.postnet") and "running_mean" in k for k in a)


def test_three_steps_in_another_process():
    a = three_steps("tf32", "flash", 4, det=True)
    env = dict(os.environ)
    r = subprocess.run([sys.executable, os.path.join(HERE, "_det_train_worker.py"), "tf32", "flash", "4"], capture_output=True, text=True,
                       timeout=900, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    assert r.stdout.strip().splitlines()[-1] == digest(a)


@pytest.mark.parametrize("prec,att", CONFIGS)
def test_one_step_agrees_with_the_default_path(prec, att):
    a = three_steps(prec, att, 0, det=True, steps=1)
    b = three_steps(prec, att, 0, det=False, steps=1)
    assert abs(float(a["loss0"]) - float(b["loss0"])) <= 1e-4 * abs(float(b["loss0"]))
    for k in a:
        if k.startswith("grad0."):
            gmax = float(b[k].abs().max())
            assert float((a[k] - b[k]).abs().max()) <= 1e-2 * gmax + 1e-6, k


def test_torch_flag_makes_the_step_deterministic():
    was = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        a = three_steps("tf32", "flash", 0, det=False, steps=2)
    finally:
        torch.use_deterministic_algorithms(was)
    b = three_steps("tf32", "flash", 0, det=True, steps=2)
    assert_equal_states(a, b)


def test_eval_loss_repeats():
    m = make_model("fp32", "materialized", 0, True).eval()
    bt = {k: v.cuda() for k, v in make_batch(4, 40, 200, seed=5, ilens=[40, 31, 17, 25], olens=[200, 150, 90, 120]).items()}
    with torch.no_grad():
        l1, r1 = m(*[bt[k] for k in KEYS])
        l2, r2 = m(*[bt[k] for k in KEYS])
    assert torch.equal(l1, l2) and r1 == r2


def test_aligner_trains_bit_for_bit():
    from _aligner_corpus import fixture_lines, render
    from fastspeech2_b200 import aligner as A
    lines = fixture_lines(64)
    sym = A.build_symbols(fixture_lines())
    corpus = A.Corpus(lines, sym, mels=render(lines, 0))
    runs = []
    for _ in range(2):
        model, hist = A.train(corpus, len(sym), steps=30, batch=16, bin_start=15, seed=0, log=lambda m: None, log_every=10, deterministic=True)
        runs.append((model.state_dict(), A.extract(model, corpus), hist))
    (s1, d1, h1), (s2, d2, h2) = runs
    assert s1.keys() == s2.keys() and all(torch.equal(s1[k], s2[k]) for k in s1)
    assert all(np.array_equal(a, b) for a, b in zip(d1, d2)) and h1 == h2


def test_profiled_kernels_hold_no_float_atomics():
    from torch.profiler import ProfilerActivity, profile
    names = set()
    for prec, att in CONFIGS:
        torch.manual_seed(0)
        m = make_model(prec, att, 4, True)
        opt = O.get_std_opt(m, 384, 100, 1.0)
        bt = {k: v.cuda() for k, v in make_batch(4, 40, 200, seed=5, ilens=[40, 31, 17, 25], olens=[200, 150, 90, 120]).items()}
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            loss, _ = m(*[bt[k] for k in KEYS], speakers=SPEAKERS.cuda())
            loss.backward()
            opt.clip_and_step(1.0)
            torch.cuda.synchronize()
        names |= {D.short_name(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    assert names & D.DEFAULT_ATOMIC == set(), sorted(names & D.DEFAULT_ATOMIC)
    assert {"colsum_kernel<true>", "scatter_group_sum_kernel", "ordered_sum_f64_kernel"} <= names
