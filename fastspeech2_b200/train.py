"""Train-mode forward + backward of `FeedForwardTransformer` (SURVEY.md section 8f-1): what
`model.train(); loss, report = model(xs, ilens, ys, olens, ds, es, ps); loss.backward()` of train_fastspeech.py:100-123 runs.

Every number is produced by kernels of libfs2b200.so (csrc/train.cu + the fp32 forward kernels); torch.autograd is used only
as the graph that chains them: each stage below is a `torch.autograd.Function` whose forward / backward are C-ABI calls.
Arithmetic is fp32 on CUDA cores by default (the reference trains in fp32); with `train_precision="tf32"` every
convolution and projection (`ConvFn`: forward, input and weight gradient) runs on the tensor cores in tf32 instead, the
way a reference user on an H100 gets TF32 for every Conv1d from cuDNN's defaults (DESIGN.md §10).  The stage order,
dropout sites and BatchNorm batch statistics follow the reference modules line by line (cited at each step of
`train_forward`).  With `train_attention="flash"` (tf32 only) self-attention runs on the fused tensor-core kernels of
csrc/attention_train_tc.cu (`FlashAttentionFn`, DESIGN.md §13) instead of the materialized `AttentionFn`.

Deterministic mode (`det=True` on the Functions below, `conv_math(math, True)` for ConvFn, DESIGN.md §26): every sum that the default kernels take with
floating-point atomics runs on the library's `_det` twins instead, which add per-CTA partials from a workspace in a fixed
order.  `train_forward` turns it on for a model built with `train_deterministic` and whenever
`torch.are_deterministic_algorithms_enabled()`; the same weights, batches and seed then give the same bits every run.

Dropout masks come from `MaskSource`: the library's Philox kernel in production, or masks injected by a test so that the
reference (with `torch.nn.functional.dropout` patched to consume the same list) and this path drop the same elements.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import List, Optional, Sequence

import torch

from . import _lib
from . import length_regulator as _lr
from ._kernel_module import query_bytes

ACT_NONE, ACT_RELU, ACT_TANH = 0, 1, 2
DET_SUMS = 0x100     # or'ed into ConvFn's `math`: its weight and bias gradients take the ordered sums (conv_math)


def _st(t: torch.Tensor) -> int:
    return _lib.stream_ptr(t.device)


def _p(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _chk(rc: int, what: str) -> None:
    _lib.check(rc, what)


def _c(t: torch.Tensor) -> torch.Tensor:
    return t if t.is_contiguous() else t.contiguous()


def _det_ws(entry: str, device, *shape):
    """(workspace, bytes) of the ordered entry `entry` for `shape` (its `_ws_bytes` query), from the caching allocator."""
    nbytes = query_bytes(entry + "_ws_bytes", *shape)
    return torch.empty((max(nbytes, 1),), dtype=torch.uint8, device=device), nbytes


def deterministic_step(model) -> bool:
    """Whether a train step of `model` sums in the fixed order of the `_det` entries: the model's `train_deterministic`,
    or torch's own flag (`torch.use_deterministic_algorithms(True)`) at the time of the step."""
    return bool(getattr(model, "train_deterministic", False)) or torch.are_deterministic_algorithms_enabled()


# ------------------------------------------------------------------------------------------------------------------------
class MaskSource:
    """Dropout masks (uint8, 1 = keep) in call order.  `injected`: a list of bool / uint8 tensors in OUR layout
    ([B, time, channel]; attention: [B, heads, L, L]) consumed in order (tests); else Philox masks from the library."""

    def __init__(self, seed: int = 0, injected: Optional[Sequence[torch.Tensor]] = None):
        self.seed, self.offset = int(seed), 0
        self.injected = list(injected) if injected is not None else None
        self.calls = 0

    def next(self, shape, p: float, device) -> torch.Tensor:
        self.calls += 1
        if self.injected is not None:
            m = self.injected.pop(0)
            if tuple(m.shape) != tuple(shape):
                raise RuntimeError(f"injected dropout mask {self.calls} has shape {tuple(m.shape)}, expected {tuple(shape)}")
            return _c(m.to(device=device, dtype=torch.uint8))
        n = 1
        for s in shape:
            n *= int(s)
        m = torch.empty(shape, dtype=torch.uint8, device=device)
        _chk(_lib.load().fs2_dropout_mask(m.data_ptr(), n, float(p), self.seed, self.offset, _lib.stream_ptr(device)), "fs2_dropout_mask")
        self.offset += (n + 3) // 4
        return m

    def attention(self, shape, p: float, device):
        """The mask source of a fused attention site: (injected mask, 0, 0), or (None, seed, offset) for the kernels to
        regenerate the Philox mask `next` would have drawn.  `offset` advances exactly as in `next`, so every later mask of
        the step is unchanged and both attention paths drop the same elements; nothing [B, h, L, L] is allocated."""
        if self.injected is not None:
            return self.next(shape, p, device), 0, 0
        self.calls += 1
        n = 1
        for s in shape:
            n *= int(s)
        off = self.offset
        self.offset += (n + 3) // 4
        return None, self.seed, off


# ------------------------------------------------------------------------------------------------------------------------
class ConvFn(torch.autograd.Function):
    """out = act(conv1d_same(x, w) + bias) (+ resid); x [B,L,K], w [N,K,taps] (nn.Conv1d) or [N,K] (nn.Linear).
    `math`: _lib.MATH_FP32 (CUDA cores) or _lib.MATH_TF32 (forward and input gradient on the tap GEMM's tf32 family,
    weight gradient on the tensor-core wgrad kernel; the bias gradient is the same column sum in both).
    `math | DET_SUMS` (conv_math): weight and bias gradients summed in a fixed order (fs2_conv_wgrad_det; tf32:
    fs2_colsum_det for the bias)."""

    @staticmethod
    def forward(ctx, x, w, bias, act, resid, math=_lib.MATH_FP32):
        lib = _lib.load()
        x = _c(x)
        B, L, K = x.shape
        N = w.shape[0]
        taps = w.shape[2] if w.dim() == 3 else 1
        assert not (act != ACT_NONE and resid is not None)
        det, math = bool(math & DET_SUMS), math & ~DET_SUMS
        if math not in (_lib.MATH_FP32, _lib.MATH_TF32):
            raise ValueError(f"ConvFn: math mode {math} is neither MATH_FP32 nor MATH_TF32")
        out = torch.empty((B, L, N), dtype=torch.float32, device=x.device)
        scratch = torch.empty((N * K * taps,), dtype=torch.float32, device=x.device)
        wc = _c(w.detach())
        args = (x.data_ptr(), B, L, K, wc.data_ptr(), _p(None if bias is None else _c(bias.detach())), N, taps, int(act),
                _p(None if resid is None else _c(resid)), out.data_ptr(), scratch.data_ptr())
        if math == _lib.MATH_FP32:
            _chk(lib.fs2_conv_forward(*args, _st(x)), "fs2_conv_forward")
        else:
            _chk(lib.fs2_conv_forward_ex(*args, math, _st(x)), "fs2_conv_forward_ex")
        ctx.save_for_backward(x, wc, out if act != ACT_NONE else None)
        ctx.meta = (B, L, K, N, taps, int(act), bias is not None, resid is not None, w.shape)
        ctx.math = math
        ctx.det = bool(det)
        return out

    @staticmethod
    def backward(ctx, dy):
        lib = _lib.load()
        x, w, out = ctx.saved_tensors
        B, L, K, N, taps, act, has_bias, has_resid, wshape = ctx.meta
        dy = _c(dy)
        g = dy
        if act != ACT_NONE:
            g = torch.empty_like(dy)
            _chk(lib.fs2_act_backward(dy.data_ptr(), out.data_ptr(), act, g.data_ptr(), dy.numel(), _st(dy)), "fs2_act_backward")
        dx = dw = db = None
        tf32 = ctx.math == _lib.MATH_TF32
        if ctx.needs_input_grad[0]:
            dx = torch.empty((B, L, K), dtype=torch.float32, device=dy.device)
            scratch = torch.empty((N * K * taps,), dtype=torch.float32, device=dy.device)
            args = (g.data_ptr(), B, L, N, w.data_ptr(), K, taps, dx.data_ptr(), scratch.data_ptr())
            if tf32:
                _chk(lib.fs2_conv_dgrad_ex(*args, ctx.math, _st(dy)), "fs2_conv_dgrad_ex")
            else:
                _chk(lib.fs2_conv_dgrad(*args, _st(dy)), "fs2_conv_dgrad")
        if ctx.needs_input_grad[1]:
            dw = torch.zeros(wshape, dtype=torch.float32, device=dy.device)
            db = torch.zeros((N,), dtype=torch.float32, device=dy.device) if has_bias else None
            if tf32:
                nbytes = wgrad_tc_ws_bytes(B, L, N, K, taps)
                ws = torch.empty((max(nbytes, 1),), dtype=torch.uint8, device=dy.device)
                _chk(lib.fs2_conv_wgrad_tc(g.data_ptr(), x.data_ptr(), B, L, N, K, taps, dw.data_ptr(), _p(None if ctx.det else db), ws.data_ptr(),
                                           nbytes, _st(dy)), "fs2_conv_wgrad_tc")
                if ctx.det and db is not None:      # the tf32 weight gradient is ordered already; its bias column sum is not
                    ws, nbytes = _det_ws("fs2_colsum_det", dy.device, B * L, N)
                    _chk(lib.fs2_colsum_det(g.data_ptr(), B * L, N, db.data_ptr(), ws.data_ptr(), nbytes, _st(dy)), "fs2_colsum_det")
            elif ctx.det:
                ws, nbytes = _det_ws("fs2_conv_wgrad_det", dy.device, B, L, N, K, taps)
                _chk(lib.fs2_conv_wgrad_det(g.data_ptr(), x.data_ptr(), B, L, N, K, taps, dw.data_ptr(), _p(db), ws.data_ptr(), nbytes, _st(dy)),
                     "fs2_conv_wgrad_det")
            else:
                _chk(lib.fs2_conv_wgrad(g.data_ptr(), x.data_ptr(), B, L, N, K, taps, dw.data_ptr(), _p(db), _st(dy)), "fs2_conv_wgrad")
        return dx, dw, db, None, (dy if has_resid else None), None


def conv_math(math: int, det: bool) -> int:
    """ConvFn's `math` argument: the math mode, with DET_SUMS when the step takes the ordered sums."""
    return math | DET_SUMS if det else math


def wgrad_tc_ws_bytes(B: int, L: int, N: int, K: int, taps: int) -> int:
    """Workspace bytes of fs2_conv_wgrad_tc for this shape (raises on a size the library rejects)."""
    n = C.c_size_t(0)
    _chk(_lib.load().fs2_conv_wgrad_tc_ws_bytes(int(B), int(L), int(N), int(K), int(taps), C.byref(n)), "fs2_conv_wgrad_tc_ws_bytes")
    return int(n.value)


class LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, eps, det=False):
        lib = _lib.load()
        x = _c(x)
        C_ = x.shape[-1]
        rows = x.numel() // C_
        out = torch.empty_like(x)
        _chk(lib.fs2_op_layernorm(x.data_ptr(), None, _c(gamma.detach()).data_ptr(), _c(beta.detach()).data_ptr(), float(eps), rows, C_, out.data_ptr(),
                                  _st(x)), "fs2_op_layernorm")
        ctx.save_for_backward(x, gamma.detach())
        ctx.eps = float(eps)
        ctx.det = bool(det)
        return out

    @staticmethod
    def backward(ctx, dy):
        lib = _lib.load()
        x, gamma = ctx.saved_tensors
        dy = _c(dy)
        C_ = x.shape[-1]
        rows = x.numel() // C_
        dx = torch.empty_like(x)
        dg = torch.zeros((C_,), dtype=torch.float32, device=x.device)
        db = torch.zeros((C_,), dtype=torch.float32, device=x.device)
        args = (x.data_ptr(), dy.data_ptr(), _c(gamma).data_ptr(), ctx.eps, rows, C_, dx.data_ptr(), dg.data_ptr(), db.data_ptr())
        if ctx.det:
            ws, nbytes = _det_ws("fs2_layernorm_backward_det", x.device, rows, C_)
            _chk(lib.fs2_layernorm_backward_det(*args, ws.data_ptr(), nbytes, _st(x)), "fs2_layernorm_backward_det")
        else:
            _chk(lib.fs2_layernorm_backward(*args, _st(x)), "fs2_layernorm_backward")
        return dx, dg, db, None, None


class AddFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        a, b = _c(a), _c(b)
        out = torch.empty_like(a)
        _chk(_lib.load().fs2_add(a.data_ptr(), b.data_ptr(), out.data_ptr(), a.numel(), _st(a)), "fs2_add")
        return out

    @staticmethod
    def backward(ctx, dy):
        return dy, dy


class DropoutFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, mask, p):
        x = _c(x)
        out = torch.empty_like(x)
        _chk(_lib.load().fs2_dropout_apply(x.data_ptr(), mask.data_ptr(), float(p), out.data_ptr(), x.numel(), _st(x)), "fs2_dropout_apply")
        ctx.save_for_backward(mask)
        ctx.p = float(p)
        return out

    @staticmethod
    def backward(ctx, dy):
        (mask,) = ctx.saved_tensors
        dy = _c(dy)
        dx = torch.empty_like(dy)
        _chk(_lib.load().fs2_dropout_apply(dy.data_ptr(), mask.data_ptr(), ctx.p, dx.data_ptr(), dy.numel(), _st(dy)), "fs2_dropout_apply")
        return dx, None, None


class ReluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = _c(x)
        y = torch.empty_like(x)
        _chk(_lib.load().fs2_relu(x.data_ptr(), y.data_ptr(), x.numel(), _st(x)), "fs2_relu")
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        dy = _c(dy)
        dx = torch.empty_like(dy)
        _chk(_lib.load().fs2_act_backward(dy.data_ptr(), y.data_ptr(), ACT_RELU, dx.data_ptr(), dy.numel(), _st(dy)), "fs2_act_backward")
        return dx


def _bgemm(a, a_str, b, b_str, c, c_str, batch, heads, M, N, K, alpha, st):
    _chk(_lib.load().fs2_bgemm(a, *a_str, b, *b_str, c, *c_str, batch, heads, M, N, K, float(alpha), st), "fs2_bgemm")


class AttentionFn(torch.autograd.Function):
    """core/attention.py:52-73 on q, k, v [B, L, C] (heads contiguous): scores, mask, softmax, masked_fill, dropout, P.V."""

    @staticmethod
    def forward(ctx, q, k, v, lens, heads, p_drop, dmask):
        q, k, v = _c(q), _c(k), _c(v)
        B, L, C_ = q.shape
        dk = C_ // heads
        st = _st(q)
        lib = _lib.load()
        s = torch.empty((B, heads, L, L), dtype=torch.float32, device=q.device)
        qs = (L * C_, dk, C_, 1)                       # (batch, head, row, col) strides of a [L, dk] head slice
        kt = (L * C_, dk, 1, C_)                       # K^T: rows = d, cols = key
        ss = (heads * L * L, L * L, L, 1)
        _bgemm(q.data_ptr(), qs, k.data_ptr(), kt, s.data_ptr(), ss, B, heads, L, L, dk, 1.0 / math.sqrt(dk), st)
        p = torch.empty_like(s)
        pd = torch.empty_like(s)
        _chk(lib.fs2_attn_softmax(s.data_ptr(), _p(lens), _p(dmask), float(p_drop), B, heads, L, p.data_ptr(), pd.data_ptr(), st), "fs2_attn_softmax")
        ctxv = torch.empty((B, L, C_), dtype=torch.float32, device=q.device)
        _bgemm(pd.data_ptr(), ss, v.data_ptr(), qs, ctxv.data_ptr(), qs, B, heads, L, dk, L, 1.0, st)
        ctx.save_for_backward(q, k, v, p, pd, dmask)
        ctx.meta = (B, L, C_, heads, float(p_drop))
        return ctxv

    @staticmethod
    def backward(ctx, dctx):
        q, k, v, p, pd, dmask = ctx.saved_tensors
        B, L, C_, heads, p_drop = ctx.meta
        dk = C_ // heads
        dctx = _c(dctx)
        st = _st(dctx)
        lib = _lib.load()
        qs = (L * C_, dk, C_, 1)
        qt = (L * C_, dk, 1, C_)
        ss = (heads * L * L, L * L, L, 1)
        st_t = (heads * L * L, L * L, 1, L)            # transposed view of a [L, L] score matrix
        dv = torch.empty_like(v)
        _bgemm(pd.data_ptr(), st_t, dctx.data_ptr(), qs, dv.data_ptr(), qs, B, heads, L, dk, L, 1.0, st)          # dV = Pd^T dO
        dpd = torch.empty_like(p)
        _bgemm(dctx.data_ptr(), qs, v.data_ptr(), qt, dpd.data_ptr(), ss, B, heads, L, L, dk, 1.0, st)           # dPd = dO V^T
        ds = torch.empty_like(p)
        _chk(lib.fs2_attn_softmax_backward(p.data_ptr(), dpd.data_ptr(), _p(dmask), p_drop, B, heads, L, ds.data_ptr(), st), "fs2_attn_softmax_backward")
        scale = 1.0 / math.sqrt(dk)
        dq = torch.empty_like(q)
        dkk = torch.empty_like(k)
        _bgemm(ds.data_ptr(), ss, k.data_ptr(), qs, dq.data_ptr(), qs, B, heads, L, dk, L, scale, st)            # dQ = dS K / sqrt(dk)
        _bgemm(ds.data_ptr(), st_t, q.data_ptr(), qs, dkk.data_ptr(), qs, B, heads, L, dk, L, scale, st)         # dK = dS^T Q / sqrt(dk)
        return dq, dkk, dv, None, None, None, None


def attn_train_ws_bytes(B: int, L: int, C_: int, heads: int) -> int:
    """Workspace bytes of fs2_attn_train_forward / _backward for this shape (raises on a shape the library rejects)."""
    n = C.c_size_t(0)
    _chk(_lib.load().fs2_attn_train_ws_bytes(int(B), int(L), int(C_), int(heads), C.byref(n)), "fs2_attn_train_ws_bytes")
    return int(n.value)


class FlashAttentionFn(torch.autograd.Function):
    """AttentionFn's contract on the fused tf32 kernels (DESIGN.md §13): saves q, k, v, O and the row log-sum-exp only;
    the dropout mask is `dmask` (injected) or regenerated from (seed, offset)."""

    @staticmethod
    def forward(ctx, q, k, v, lens, heads, p_drop, dmask, seed, offset):
        q, k, v = _c(q), _c(k), _c(v)
        B, L, C_ = q.shape
        nbytes = attn_train_ws_bytes(B, L, C_, heads)
        ws = torch.empty((nbytes,), dtype=torch.uint8, device=q.device)
        out = torch.empty((B, L, C_), dtype=torch.float32, device=q.device)
        lse = torch.empty((B * heads, L), dtype=torch.float32, device=q.device)
        _chk(_lib.load().fs2_attn_train_forward(q.data_ptr(), k.data_ptr(), v.data_ptr(), lens.data_ptr(), B, L, C_, heads, float(p_drop), _p(dmask),
                                                int(seed), int(offset), out.data_ptr(), lse.data_ptr(), ws.data_ptr(), nbytes, _st(q)),
             "fs2_attn_train_forward")
        ctx.save_for_backward(q, k, v, out, lse, lens, dmask)
        ctx.meta = (heads, float(p_drop), int(seed), int(offset))
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, out, lse, lens, dmask = ctx.saved_tensors
        heads, p_drop, seed, offset = ctx.meta
        dout = _c(dout)
        B, L, C_ = q.shape
        nbytes = attn_train_ws_bytes(B, L, C_, heads)
        ws = torch.empty((nbytes,), dtype=torch.uint8, device=q.device)
        dq, dkk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        _chk(_lib.load().fs2_attn_train_backward(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(), dout.data_ptr(),
                                                 lens.data_ptr(), B, L, C_, heads, p_drop, _p(dmask), seed, offset, dq.data_ptr(), dkk.data_ptr(),
                                                 dv.data_ptr(), ws.data_ptr(), nbytes, _st(dout)), "fs2_attn_train_backward")
        return dq, dkk, dv, None, None, None, None, None, None


class EmbedFn(torch.autograd.Function):
    """nn.Embedding(padding_idx=0) + x + alpha * pe (fastspeech.py:65-67, embedding.py:105-120, before its dropout)."""

    @staticmethod
    def forward(ctx, xs, table, alpha, pe, det=False):
        B, T = xs.shape
        C_ = table.shape[1]
        out = torch.empty((B, T, C_), dtype=torch.float32, device=xs.device)
        pe2 = _c(pe.reshape(-1, C_))
        _chk(_lib.load().fs2_embed_posenc(xs.data_ptr(), _c(table.detach()).data_ptr(), table.shape[0], pe2.data_ptr(), alpha.detach().reshape(1).data_ptr(),
                                          B, T, C_, out.data_ptr(), None, None, _st(xs)), "fs2_embed_posenc")
        ctx.save_for_backward(xs, pe2)
        ctx.meta = (B, T, C_, table.shape[0])
        ctx.det = bool(det)
        return out

    @staticmethod
    def backward(ctx, dy):
        xs, pe2 = ctx.saved_tensors
        B, T, C_, n_sym = ctx.meta
        dy = _c(dy)
        dtab = torch.zeros((n_sym, C_), dtype=torch.float32, device=dy.device)
        dalpha = torch.zeros((1,), dtype=torch.float32, device=dy.device)
        args = (xs.data_ptr(), dy.data_ptr(), pe2.data_ptr(), B, T, C_, n_sym, dtab.data_ptr(), dalpha.data_ptr())
        if ctx.det:
            ws, nbytes = _det_ws("fs2_embed_backward_det", dy.device, B, T, C_, n_sym)
            _chk(_lib.load().fs2_embed_backward_det(*args, ws.data_ptr(), nbytes, _st(dy)), "fs2_embed_backward_det")
        else:
            _chk(_lib.load().fs2_embed_backward(*args, _st(dy)), "fs2_embed_backward")
        return None, dtab, dalpha.reshape(()), None, None


class PosEncFn(torch.autograd.Function):
    """x + alpha * pe[:T] (ScaledPositionalEncoding of the decoder input layer, before its dropout)."""

    @staticmethod
    def forward(ctx, x, alpha, pe, det=False):
        x = _c(x)
        B, T, C_ = x.shape
        pe2 = _c(pe.reshape(-1, C_))
        out = torch.empty_like(x)
        _chk(_lib.load().fs2_posenc_add(x.data_ptr(), pe2.data_ptr(), alpha.detach().reshape(1).data_ptr(), B, T, C_, out.data_ptr(), _st(x)), "fs2_posenc_add")
        ctx.save_for_backward(pe2)
        ctx.meta = (B, T, C_)
        ctx.det = bool(det)
        return out

    @staticmethod
    def backward(ctx, dy):
        (pe2,) = ctx.saved_tensors
        B, T, C_ = ctx.meta
        dy = _c(dy)
        dalpha = torch.zeros((1,), dtype=torch.float32, device=dy.device)
        args = (None, dy.data_ptr(), pe2.data_ptr(), B, T, C_, 0, None, dalpha.data_ptr())
        if ctx.det:
            ws, nbytes = _det_ws("fs2_embed_backward_det", dy.device, B, T, C_, 0)
            _chk(_lib.load().fs2_embed_backward_det(*args, ws.data_ptr(), nbytes, _st(dy)), "fs2_embed_backward_det")
        else:
            _chk(_lib.load().fs2_embed_backward(*args, _st(dy)), "fs2_embed_backward")
        return dy, dalpha.reshape(()), None, None


class RowDotFn(torch.autograd.Function):
    """Linear(C -> 1).squeeze(-1), masked_fill(pad, 0): the predictors' heads."""

    @staticmethod
    def forward(ctx, x, w, bias, lens, det=False):
        x = _c(x)
        B, L, C_ = x.shape
        y = torch.empty((B, L), dtype=torch.float32, device=x.device)
        wv = _c(w.detach().reshape(-1))
        _chk(_lib.load().fs2_rowdot(x.data_ptr(), wv.data_ptr(), _c(bias.detach()).data_ptr(), _p(lens), B * L, L, C_, y.data_ptr(), _st(x)), "fs2_rowdot")
        ctx.save_for_backward(x, wv, lens)
        ctx.wshape = w.shape
        ctx.det = bool(det)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, wv, lens = ctx.saved_tensors
        B, L, C_ = x.shape
        dy = _c(dy)
        dx = torch.empty_like(x)
        dw = torch.zeros((C_,), dtype=torch.float32, device=x.device)
        db = torch.zeros((1,), dtype=torch.float32, device=x.device)
        args = (x.data_ptr(), wv.data_ptr(), dy.data_ptr(), _p(lens), B * L, L, C_, dx.data_ptr(), dw.data_ptr(), db.data_ptr())
        if ctx.det:
            ws, nbytes = _det_ws("fs2_rowdot_backward_det", x.device, B * L, C_)
            _chk(_lib.load().fs2_rowdot_backward_det(*args, ws.data_ptr(), nbytes, _st(x)), "fs2_rowdot_backward_det")
        else:
            _chk(_lib.load().fs2_rowdot_backward(*args, _st(x)), "fs2_rowdot_backward")
        return dx, dw.reshape(ctx.wshape), db, None, None


class SpeakerAddFn(torch.autograd.Function):
    """hs + E[spk].unsqueeze(1) over every row t < T (DESIGN.md section 25); E [n, C].  The table's gradient comes from the
    deterministic fs2_speaker_add_backward (per-utterance column sums, then one ordered sum per speaker, no atomics)."""

    @staticmethod
    def forward(ctx, x, spk, table):
        x = _c(x)
        B, T, C_ = x.shape
        out = torch.empty_like(x)
        _chk(_lib.load().fs2_speaker_add(x.data_ptr(), spk.data_ptr(), _c(table.detach()).data_ptr(), B, T, C_, table.shape[0], out.data_ptr(),
                                         _st(x)), "fs2_speaker_add")
        ctx.save_for_backward(spk)
        ctx.meta = (B, T, C_, table.shape[0])
        return out

    @staticmethod
    def backward(ctx, dy):
        (spk,) = ctx.saved_tensors
        B, T, C_, n = ctx.meta
        dy = _c(dy)
        dtab = torch.zeros((n, C_), dtype=torch.float32, device=dy.device)
        nbytes = speaker_add_ws_bytes(B, C_)
        ws = torch.empty((max(nbytes, 1),), dtype=torch.uint8, device=dy.device)
        _chk(_lib.load().fs2_speaker_add_backward(dy.data_ptr(), spk.data_ptr(), B, T, C_, n, dtab.data_ptr(), ws.data_ptr(), nbytes, _st(dy)),
             "fs2_speaker_add_backward")
        return dy, None, dtab


class SpembAddFn(torch.autograd.Function):
    """hs + v.unsqueeze(1) over every row t < T, v = W . normalize(e) + bias the projected speaker embeddings (DESIGN.md
    section 27; `spemb_project` computes v and the normalised e).  The add is fs2_speaker_add with ids 0 .. B-1 and v as
    the table, one fp32 add.  Backward: dv[b] = sum_t dy[b, t] (fs2_speaker_add_backward with those ids, a fixed tree
    order), then fs2_spemb_project_backward: dW += sum_b dv[b] (x) e_hat[b], dbias += sum_b dv[b], b ascending.  No
    atomics, so it is deterministic in every train mode.  The embeddings get no gradient."""

    @staticmethod
    def forward(ctx, x, v, en, weight, bias):
        x = _c(x)
        B, T, C_ = x.shape
        ids = torch.arange(B, dtype=torch.int64, device=x.device)
        out = torch.empty_like(x)
        _chk(_lib.load().fs2_speaker_add(x.data_ptr(), ids.data_ptr(), v.data_ptr(), B, T, C_, max(B, 1), out.data_ptr(), _st(x)),
             "fs2_speaker_add")
        ctx.save_for_backward(ids, en)
        ctx.meta = (B, T, C_, int(en.shape[1]))
        return out

    @staticmethod
    def backward(ctx, dy):
        ids, en = ctx.saved_tensors
        B, T, C_, D = ctx.meta
        dy = _c(dy)
        lib = _lib.load()
        dv = torch.zeros((B, C_), dtype=torch.float32, device=dy.device)
        nbytes = speaker_add_ws_bytes(B, C_)
        ws = torch.empty((max(nbytes, 1),), dtype=torch.uint8, device=dy.device)
        _chk(lib.fs2_speaker_add_backward(dy.data_ptr(), ids.data_ptr(), B, T, C_, max(B, 1), dv.data_ptr(), ws.data_ptr(), nbytes,
                                          _st(dy)), "fs2_speaker_add_backward")
        dW = torch.zeros((C_, D), dtype=torch.float32, device=dy.device)
        db = torch.zeros((C_,), dtype=torch.float32, device=dy.device)
        _chk(lib.fs2_spemb_project_backward(dv.data_ptr(), en.data_ptr(), B, D, C_, dW.data_ptr(), db.data_ptr(), _st(dy)),
             "fs2_spemb_project_backward")
        return dy, None, None, dW, db


def spemb_project(weight: torch.Tensor, bias: torch.Tensor, spembs: torch.Tensor):
    """fs2_spemb_project: (v [B, adim], e_hat [B, D], status [1] int32) for float32 [B, D] embeddings on the device.
    status has FS2_SPEMB_NONFINITE set when some embedding holds a non-finite value or its fp32 sum of squares overflows."""
    B, D = spembs.shape
    A = int(weight.shape[0])
    dev = spembs.device
    v = torch.empty((B, A), dtype=torch.float32, device=dev)
    en = torch.empty((B, D), dtype=torch.float32, device=dev)
    status = torch.zeros((1,), dtype=torch.int32, device=dev)
    _chk(_lib.load().fs2_spemb_project(_c(weight.detach()).data_ptr(), _c(bias.detach()).data_ptr(), _c(spembs).data_ptr(), B, D, A,
                                       v.data_ptr(), en.data_ptr(), None, status.data_ptr(), _st(spembs)), "fs2_spemb_project")
    return v, en, status


def speaker_add_ws_bytes(B: int, C_: int) -> int:
    """Workspace bytes of fs2_speaker_add_backward for B utterances of C channels."""
    n = C.c_size_t(0)
    _chk(_lib.load().fs2_speaker_add_backward_ws_bytes(int(B), int(C_), C.byref(n)), "fs2_speaker_add_backward_ws_bytes")
    return int(n.value)


class LengthRegulatorFn(torch.autograd.Function):
    """length_regulator.py:38-95 with the ground-truth durations; backward = per-phoneme sum of its frames' gradients."""

    @staticmethod
    def forward(ctx, hs, ds, ilens, L):
        hs = _c(hs)
        cum, _, stats, il = _lr.plan(hs, ds, ilens, 1.0)
        out = _lr.gather(hs, cum, il, int(L))
        ctx.save_for_backward(cum, il)
        ctx.meta = (hs.shape, int(L))
        ctx.stats = stats
        return out

    @staticmethod
    def backward(ctx, dy):
        cum, il = ctx.saved_tensors
        (B, T, C_), L = ctx.meta
        dy = _c(dy)
        dhs = torch.empty((B, T, C_), dtype=torch.float32, device=dy.device)
        _chk(_lib.load().fs2_length_regulator_backward(dy.data_ptr(), cum.data_ptr(), il.data_ptr(), B, T, C_, L, dhs.data_ptr(), _st(dy)),
             "fs2_length_regulator_backward")
        return dhs, None, None, None


class OneHotLinearAddFn(torch.autograd.Function):
    """hs + Linear(n_bins -> C)(one_hot(ids)) (fastspeech.py:218-219); W [C, n_bins], b [C]."""

    @staticmethod
    def forward(ctx, x, ids, W, b, det=False):
        x = _c(x)
        rows, C_ = x.numel() // x.shape[-1], x.shape[-1]
        out = torch.empty_like(x)
        _chk(_lib.load().fs2_onehot_linear_forward(x.data_ptr(), ids.data_ptr(), _c(W.detach()).data_ptr(), _c(b.detach()).data_ptr(), rows, C_, W.shape[1],
                                                   out.data_ptr(), _st(x)), "fs2_onehot_linear_forward")
        ctx.save_for_backward(ids)
        ctx.meta = (rows, C_, W.shape[1])
        ctx.det = bool(det)
        return out

    @staticmethod
    def backward(ctx, dy):
        (ids,) = ctx.saved_tensors
        rows, C_, nb = ctx.meta
        dy = _c(dy)
        dW = torch.zeros((C_, nb), dtype=torch.float32, device=dy.device)
        db = torch.zeros((C_,), dtype=torch.float32, device=dy.device)
        args = (ids.data_ptr(), dy.data_ptr(), rows, C_, nb, dW.data_ptr(), db.data_ptr())
        if ctx.det:
            ws, nbytes = _det_ws("fs2_onehot_linear_backward_det", dy.device, rows, C_, nb)
            _chk(_lib.load().fs2_onehot_linear_backward_det(*args, ws.data_ptr(), nbytes, _st(dy)), "fs2_onehot_linear_backward_det")
        else:
            _chk(_lib.load().fs2_onehot_linear_backward(*args, _st(dy)), "fs2_onehot_linear_backward")
        return dy, None, dW, db, None


class BatchNormFn(torch.autograd.Function):
    """BatchNorm1d in train mode over all B*L rows of a channel (+ optional tanh); updates the running statistics."""

    @staticmethod
    def forward(ctx, x, gamma, beta, running_mean, running_var, eps, momentum, act, det=False):
        x = _c(x)
        C_ = x.shape[-1]
        rows = x.numel() // C_
        y = torch.empty_like(x)
        stats = torch.empty((2 * C_,), dtype=torch.float32, device=x.device)
        args = (x.data_ptr(), rows, C_, _c(gamma.detach()).data_ptr(), _c(beta.detach()).data_ptr(), float(eps), float(momentum), int(act),
                running_mean.data_ptr(), running_var.data_ptr(), stats.data_ptr(), y.data_ptr())
        if det:
            ws, nbytes = _det_ws("fs2_batchnorm_train_det", x.device, rows, C_)
            _chk(_lib.load().fs2_batchnorm_train_det(*args, ws.data_ptr(), nbytes, _st(x)), "fs2_batchnorm_train_det")
        else:
            scratch = torch.empty((4 * C_,), dtype=torch.float64, device=x.device)
            _chk(_lib.load().fs2_batchnorm_train(*args, scratch.data_ptr(), _st(x)), "fs2_batchnorm_train")
        ctx.save_for_backward(x, stats, gamma.detach(), y if act != ACT_NONE else None)
        ctx.meta = (rows, C_, float(eps), int(act))
        ctx.det = bool(det)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, stats, gamma, y = ctx.saved_tensors
        rows, C_, eps, act = ctx.meta
        lib = _lib.load()
        dy = _c(dy)
        g = dy
        if act != ACT_NONE:
            g = torch.empty_like(dy)
            _chk(lib.fs2_act_backward(dy.data_ptr(), y.data_ptr(), act, g.data_ptr(), dy.numel(), _st(dy)), "fs2_act_backward")
        dx = torch.empty_like(x)
        dg = torch.zeros((C_,), dtype=torch.float32, device=x.device)
        db = torch.zeros((C_,), dtype=torch.float32, device=x.device)
        args = (x.data_ptr(), g.data_ptr(), stats.data_ptr(), _c(gamma).data_ptr(), eps, rows, C_, dx.data_ptr(), dg.data_ptr(), db.data_ptr())
        if ctx.det:
            ws, nbytes = _det_ws("fs2_batchnorm_backward_det", x.device, rows, C_)
            _chk(lib.fs2_batchnorm_backward_det(*args, ws.data_ptr(), nbytes, _st(x)), "fs2_batchnorm_backward_det")
        else:
            scratch = torch.empty((4 * C_,), dtype=torch.float64, device=x.device)
            _chk(lib.fs2_batchnorm_backward(*args, scratch.data_ptr(), _st(x)), "fs2_batchnorm_backward")
        return dx, dg, db, None, None, None, None, None, None


class LossFn(torch.autograd.Function):
    """fastspeech.py:277-324 (use_masking): returns the 7 report values [l1, before, after, duration, energy, pitch, total];
    differentiable through element 6 only (the scalar the training loop back-propagates)."""

    @staticmethod
    def forward(ctx, before, after, d_outs, e_outs, p_outs, ys, ds, es, ps, ilens, olens, det=False):
        before, after, d_outs, e_outs, p_outs = (_c(t) for t in (before, after, d_outs, e_outs, p_outs))
        out7 = masked_losses(before, after, d_outs, e_outs, p_outs, ys, ds, es, ps, ilens, olens, det)
        ctx.save_for_backward(before, after, d_outs, e_outs, p_outs, ys, ds, es, ps, ilens, olens)
        return out7

    @staticmethod
    def backward(ctx, g7):
        before, after, d_outs, e_outs, p_outs, ys, ds, es, ps, ilens, olens = ctx.saved_tensors
        lib = _lib.load()
        B, L, odim = before.shape
        T = d_outs.shape[1]
        g = _c(g7[6:7].to(torch.float32))
        gb, ga = torch.empty_like(before), torch.empty_like(after)
        gd, ge, gp = torch.empty_like(d_outs), torch.empty_like(e_outs), torch.empty_like(p_outs)
        _chk(lib.fs2_loss_backward(before.data_ptr(), after.data_ptr(), ys.data_ptr(), int(ys.shape[1]), d_outs.data_ptr(), ds.data_ptr(), _lib.dur_dtype(ds),
                                   e_outs.data_ptr(), p_outs.data_ptr(), es.data_ptr(), ps.data_ptr(), ilens.data_ptr(), olens.data_ptr(), B, T, L, odim,
                                   g.data_ptr(), gb.data_ptr(), ga.data_ptr(), gd.data_ptr(), ge.data_ptr(), gp.data_ptr(), _st(before)), "fs2_loss_backward")
        return gb, ga, gd, ge, gp, None, None, None, None, None, None, None


def masked_losses(before, after, d_outs, e_outs, p_outs, ys, ds, es, ps, ilens, olens, det: bool = False) -> torch.Tensor:
    """The 7 report values of fs2_masked_losses (contiguous CUDA inputs, ys [B, >= L, odim]); `det`: fs2_masked_losses_det,
    whose five sums are added in a fixed order."""
    lib = _lib.load()
    B, L, odim = before.shape
    T = d_outs.shape[1]
    out7 = torch.empty((7,), dtype=torch.float32, device=before.device)
    args = (before.data_ptr(), after.data_ptr(), ys.data_ptr(), int(ys.shape[1]), d_outs.data_ptr(), ds.data_ptr(), _lib.dur_dtype(ds),
            e_outs.data_ptr(), p_outs.data_ptr(), es.data_ptr(), ps.data_ptr(), ilens.data_ptr(), olens.data_ptr(), B, T, L, odim, out7.data_ptr())
    if det:
        ws, nbytes = _det_ws("fs2_masked_losses_det", before.device, B, T, L, odim)
        _chk(lib.fs2_masked_losses_det(*args, ws.data_ptr(), nbytes, _st(before)), "fs2_masked_losses_det")
    else:
        scratch = torch.empty((16,), dtype=torch.float64, device=before.device)
        _chk(lib.fs2_masked_losses(*args, scratch.data_ptr(), _st(before)), "fs2_masked_losses")
    return out7


# ------------------------------------------------------------------------------------------------------------------------
def _drop(x: torch.Tensor, p: float, masks: MaskSource, channel_first: bool = False) -> torch.Tensor:
    """nn.Dropout(p) in train mode.  `channel_first`: the reference applies this dropout to a [B, C, time] tensor (conv
    stacks); injected masks arrive in our [B, time, C] layout either way (tests permute them), Philox masks have no layout."""
    if p <= 0.0:
        return x
    return DropoutFn.apply(x, masks.next(tuple(x.shape), p, x.device), p)


def _fft_blocks(stack, x, lens, heads: int, rate: float, masks: MaskSource, math: int = _lib.MATH_FP32, flash: bool = False,
                det: bool = False):
    """core/encoder.py:46-71 (post-LN, concat_after=False) x num_blocks.  `flash`: attention on the fused tf32 kernels
    (FlashAttentionFn) instead of the materialized AttentionFn.  `det`: the ordered sums of the deterministic mode."""
    B, L, C_ = x.shape
    cm = conv_math(math, det)
    for blk in stack.encoders_:
        a = blk.self_attn
        q = ConvFn.apply(x, a.linear_q.weight, a.linear_q.bias, ACT_NONE, None, cm)   # attention.py:48-50
        k = ConvFn.apply(x, a.linear_k.weight, a.linear_k.bias, ACT_NONE, None, cm)
        v = ConvFn.apply(x, a.linear_v.weight, a.linear_v.bias, ACT_NONE, None, cm)
        if flash:
            dmask, seed, off = masks.attention((B, heads, L, L), rate, x.device) if rate > 0 else (None, 0, 0)   # attention.py:69
            ctx = FlashAttentionFn.apply(q, k, v, lens, heads, rate, dmask, seed, off)
        else:
            dmask = masks.next((B, heads, L, L), rate, x.device) if rate > 0 else None       # attention.py:69
            ctx = AttentionFn.apply(q, k, v, lens, heads, rate, dmask)
        att = ConvFn.apply(ctx, a.linear_out.weight, a.linear_out.bias, ACT_NONE, None, cm)   # attention.py:74
        x = AddFn.apply(x, _drop(att, rate, masks))                                           # encoder.py:60
        x = LayerNormFn.apply(x, blk.norm1.weight, blk.norm1.bias, blk.norm1.eps, det)        # encoder.py:62
        f = blk.feed_forward
        h = ConvFn.apply(x, f.w_1.weight, f.w_1.bias, ACT_RELU, None, cm)              # modules.py:247
        h = _drop(h, rate, masks)                                                             # modules.py:248
        y = ConvFn.apply(h, f.w_2.weight, f.w_2.bias, ACT_NONE, None, cm)
        x = AddFn.apply(x, _drop(y, rate, masks))                                             # encoder.py:67
        x = LayerNormFn.apply(x, blk.norm2.weight, blk.norm2.bias, blk.norm2.eps, det)        # encoder.py:69
    return x


def _predictor(pred, x, lens, rate: float, masks: MaskSource, math: int = _lib.MATH_FP32, det: bool = False):
    """duration_predictor.py:64-86 / variance_predictor.py:39-78: [conv -> ReLU -> LayerNorm(channels) -> Dropout] x n, Linear -> 1, mask."""
    cm = conv_math(math, det)
    for layer in pred.conv:
        conv, ln = layer[0], layer[2].layer_norm
        x = ConvFn.apply(x, conv.weight, conv.bias, ACT_RELU, None, cm)
        x = LayerNormFn.apply(x, ln.weight, ln.bias, ln.eps, det)
        x = _drop(x, rate, masks, channel_first=True)
    return RowDotFn.apply(x, pred.linear.weight, pred.linear.bias, lens, det)


def train_forward(model, xs, ilens, ys, olens, ds, es, ps, masks: Optional[MaskSource] = None, speakers=None, spembs=None):
    """`FeedForwardTransformer.forward` in train mode (fastspeech.py:245-337 -> _forward :169-243).  Returns
    (loss 0-d tensor attached to the autograd graph, report_keys).  `speakers`: int64 [B] ids of a multi-speaker model;
    `spembs`: float32 [B, D] speaker embeddings of a model with spk_embed_dim = D."""
    from .fastspeech import _check_spemb_status, _check_speaker_range, _spemb_tensor, _speaker_ids, _speaker_violations
    lib = _lib.load()
    dev = xs.device
    if dev.type != "cuda":
        raise _lib.Fs2Error("train-mode forward needs CUDA tensors (no CPU fallback)")
    masks = masks or MaskSource(seed=int(torch.initial_seed()) & 0xFFFFFFFF)
    math = _lib.MATH_TF32 if model.train_precision == "tf32" else _lib.MATH_FP32
    flash = model.train_attention == "flash"
    det = deterministic_step(model)
    cm = conv_math(math, det)
    d = model.dims
    ilens = ilens.to(device=dev, dtype=torch.int64).contiguous()
    olens = olens.to(device=dev, dtype=torch.int64).contiguous()
    spk = _speaker_ids(model.n_speakers, speakers, int(xs.shape[0]), dev)
    spe = _spemb_tensor(model.spk_embed_dim, spembs, int(xs.shape[0]), dev)
    if spe is not None:     # projected first, so that its status word rides in the host read below
        proj = model.spk_embed_proj
        spe_v, spe_en, spe_status = spemb_project(proj.weight, proj.bias, spe)
    if spk is None and spe is None:
        tmax, lmax = torch.stack([ilens.max(), olens.max()]).tolist()
    else:       # the speaker range and the embeddings' status word ride in the same host read
        words = [torch.stack([ilens.max(), olens.max()])]
        if spk is not None:
            words.append(_speaker_violations(spk, model.n_speakers))
        if spe is not None:
            words.append(spe_status.to(torch.int64))
        vals = torch.cat(words).tolist()
        tmax, lmax = vals[:2]
        if spe is not None:
            _check_spemb_status(vals.pop())
        if spk is not None:
            _check_speaker_range(vals[2], model.n_speakers)
    xs = xs[:, :tmax].to(torch.int64).contiguous()                                            # fastspeech.py:266-267
    ds = ds[:, :tmax].contiguous()
    es = es[:, :lmax].to(torch.float32).contiguous()
    ps = ps[:, :lmax].to(torch.float32).contiguous()
    ys = ys.to(dtype=torch.float32, device=dev).contiguous()
    B, T = xs.shape
    L = int(lmax)
    model._extend_pe(model.encoder, T)
    model._extend_pe(model.decoder, L)
    ER, DR, PR, POST = 0.2, 0.2, 0.5, float(model.postnet_dropout_rate)                        # fastspeech.py:75-77,127-129; predictors: hp / default 0.5

    # encoder (fastspeech.py:180-184): Embedding + scaled positional encoding + dropout, FFT blocks
    enc_pos = model.encoder.embed[-1]
    x = EmbedFn.apply(xs, model.encoder.embed[0].weight, enc_pos.alpha, enc_pos.pe, det)
    x = _drop(x, ER, masks)                                                                   # embedding.py:120
    hs = _fft_blocks(model.encoder, x, ilens, d.aheads, ER, masks, math, flash, det)
    if spk is not None:     # hs + E[spk] at every row, fp32 in both train precisions
        hs = SpeakerAddFn.apply(hs, spk, model.speaker_embed.weight)
    if spe is not None:     # (hs + E[spk]) + v at every row, fp32 in both train precisions
        hs = SpembAddFn.apply(hs, spe_v, spe_en, model.spk_embed_proj.weight, model.spk_embed_proj.bias)
    # duration predictor on the encoder states, then LengthRegulator with the ground-truth durations (:209-211)
    d_outs = _predictor(model.duration_predictor, hs, ilens, model.duration_dropout_rate, masks, math, det)
    hm = LengthRegulatorFn.apply(hs, ds, ilens, L)
    e_outs = _predictor(model.energy_predictor.predictor, hm, olens, PR, masks, math, det)          # :212-215
    p_outs = _predictor(model.pitch_predictor.predictor, hm, olens, PR, masks, math, det)
    # hs + pitch_embed(one_hot(ps)) + energy_embed(one_hot(es)) (:200-206,218-219); bucket ids from the library's bucketize
    e_ids = torch.empty((B, L), dtype=torch.int64, device=dev)
    p_ids = torch.empty((B, L), dtype=torch.int64, device=dev)
    eb, pb = model.energy_predictor.energy_bins, model.pitch_predictor.pitch_bins
    _chk(lib.fs2_bucketize(es.data_ptr(), eb.data_ptr(), eb.numel(), es.numel(), e_ids.data_ptr(), _st(es)), "fs2_bucketize")
    _chk(lib.fs2_bucketize(ps.data_ptr(), pb.data_ptr(), pb.numel(), ps.numel(), p_ids.data_ptr(), _st(ps)), "fs2_bucketize")
    hm = OneHotLinearAddFn.apply(hm, p_ids, model.pitch_embed.weight, model.pitch_embed.bias, det)
    hm = OneHotLinearAddFn.apply(hm, e_ids, model.energy_embed.weight, model.energy_embed.bias, det)
    # decoder input layer (core/encoder.py:118-125): Linear -> LayerNorm -> Dropout -> ReLU -> scaled positional encoding (+ dropout)
    emb = model.decoder.embed
    z = ConvFn.apply(hm, emb[0].weight, emb[0].bias, ACT_NONE, None, cm)
    z = LayerNormFn.apply(z, emb[1].weight, emb[1].bias, emb[1].eps, det)
    z = _drop(z, DR, masks)
    z = ReluFn.apply(z)
    z = PosEncFn.apply(z, emb[4].alpha, emb[4].pe, det)
    z = _drop(z, DR, masks)
    z = _fft_blocks(model.decoder, z, olens, d.aheads, DR, masks, math, flash, det)
    before = ConvFn.apply(z, model.feat_out.weight, model.feat_out.bias, ACT_NONE, None, cm)   # :228-230
    # Postnet (modules.py:283-359): [conv(no bias) -> BatchNorm1d(batch statistics) -> tanh -> dropout] x 4, conv -> BN -> dropout; + residual
    y = before
    n_post = len(model.postnet.postnet)
    for i, layer in enumerate(model.postnet.postnet):
        conv, bn = layer[0], layer[1]
        last = i == n_post - 1
        y = ConvFn.apply(y, conv.weight, None, ACT_NONE, None, cm)
        y = BatchNormFn.apply(y, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps, bn.momentum if bn.momentum is not None else 0.1,
                              ACT_NONE if last else ACT_TANH, det)
        with torch.no_grad():
            bn.num_batches_tracked += 1
        y = _drop(y, POST, masks, channel_first=True)
    after = AddFn.apply(before, y)                                                            # :236-238
    out7 = LossFn.apply(before, after, d_outs, e_outs, p_outs, ys, ds, es, ps, ilens, olens, det)
    vals = out7.detach().tolist()
    names = ["l1_loss", "before_loss", "after_loss", "duration_loss", "energy_loss", "pitch_loss", "loss"]
    return out7[6], [{k: v} for k, v in zip(names, vals)]
