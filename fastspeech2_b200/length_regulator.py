"""LengthRegulator with the reference's module API
(core/duration_modeling/length_regulator.py:14-95) on the H100 scan + gather kernels.

    LengthRegulator()(xs[B,T,C] f32, ds[B,T] i64|i32|f32, ilens[B] i64, alpha=1.0) -> [B, max_b sum(d), C]

Semantics kept from the reference (and pinned by tests/golden/length_regulator.npz):
durations past ilens[b] are ignored; an utterance whose durations sum to 0 is expanded with
all-ones and, when alpha == 1, the ones are written back into the caller's `ds`; alpha != 1
rescales with round-half-even on a private copy; float durations are truncated like int(d_);
a negative duration raises RuntimeError; output rows past an utterance's length are 0.
"""
from __future__ import annotations


from typing import Optional

import torch

from . import _lib


INT32_MAX = 2 ** 31 - 1   # cum is int32: a plan whose max_b olens (stats[0]) exceeds this must not be gathered


def plan(xs: torch.Tensor, ds: torch.Tensor, ilens: torch.Tensor, alpha: float = 1.0,
         alpha_v: Optional[torch.Tensor] = None, d_used: Optional[torch.Tensor] = None):
    """Scan kernel only, no host sync.  Returns (cum[B,T] i32, olens[B] i64, stats[2] i64, ilens_dev);
    stats = [max_b olens, #negative durations] stays on the device -- the caller decides when to read it.
    alpha_v: optional contiguous [B,T] float32 device tensor, one speed factor per phoneme in place of `alpha` (the
    caller's ds are then not written); d_used: optional [B,T] int64 device tensor that receives the frame counts
    actually expanded (fs2_length_plan_ex)."""
    lib = _lib.load()
    if not xs.is_cuda:
        raise _lib.Fs2Error("LengthRegulator: CUDA tensors required (no CPU fallback)")
    if xs.dtype != torch.float32:
        raise _lib.Fs2Error("LengthRegulator: xs must be float32")
    assert alpha > 0
    dev = xs.device
    B, T, _ = xs.shape
    ilens_dev = ilens.to(device=dev, dtype=torch.int64).contiguous()
    ds_work = ds if (ds.is_cuda and ds.is_contiguous() and ds.shape[1] == T) else ds.to(dev)[:, :T].contiguous()
    if ds_work.shape != (B, T):
        raise _lib.Fs2Error(f"LengthRegulator: ds shape {tuple(ds.shape)} does not cover xs {tuple(xs.shape)}")
    mutate = 1 if alpha == 1.0 and alpha_v is None else 0
    cum = torch.empty((B, T), dtype=torch.int32, device=dev)
    olens = torch.empty((B,), dtype=torch.int64, device=dev)
    stats = torch.empty((2,), dtype=torch.int64, device=dev)
    _lib.check(lib.fs2_length_plan_ex(_lib.ptr(ds_work), _lib.dur_dtype(ds_work), _lib.ptr(ilens_dev), float(alpha),
                                      _lib.ptr(alpha_v), B, T, mutate, _lib.ptr(cum), _lib.ptr(olens), _lib.ptr(stats),
                                      _lib.ptr(d_used), _lib.stream_ptr(dev)), "fs2_length_plan_ex")
    if mutate and ds_work is not ds and ds.shape == ds_work.shape:
        ds.copy_(ds_work)  # keep the reference's in-place fill visible through non-contiguous / CPU callers
    return cum, olens, stats, ilens_dev


def gather(xs: torch.Tensor, cum: torch.Tensor, ilens: torch.Tensor, out_len: int, fac_in: Optional[torch.Tensor] = None,
           fac_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Expand xs by the plan `cum`.  fac_in [2,B,T] float32 / fac_out [2,B,out_len] float32 (both or neither): per-phoneme
    factors expanded to per-frame factors in the same pass, 1.0 past each utterance's length (fs2_length_gather_ex)."""
    lib = _lib.load()
    B, T, Cc = xs.shape
    out = torch.empty((B, out_len, Cc), dtype=torch.float32, device=xs.device)
    _lib.check(lib.fs2_length_gather_ex(_lib.ptr(xs), _lib.ptr(cum), _lib.ptr(ilens), B, T, Cc, _lib.ptr(out), out_len,
                                        _lib.ptr(fac_in), _lib.ptr(fac_out), _lib.stream_ptr(xs.device)),
               "fs2_length_gather_ex")
    return out


class LengthRegulator(torch.nn.Module):
    """Drop-in for core.duration_modeling.length_regulator.LengthRegulator."""

    def __init__(self, pad_value: float = 0.0):
        super().__init__()
        if pad_value != 0.0:
            raise ValueError("only pad_value=0.0 is supported (the reference always pads with 0.0, length_regulator.py:65)")
        self.pad_value = pad_value

    def forward(self, xs: torch.Tensor, ds: torch.Tensor, ilens: torch.Tensor, alpha: float = 1.0) -> torch.Tensor:
        if xs.is_cuda and torch.cuda.current_device() != (xs.device.index or 0):
            with torch.cuda.device(xs.device):      # the kernels run on the current device: select the data's
                return self.forward(xs, ds, ilens, alpha)
        cum, _, stats, ilens_dev = plan(xs, ds, ilens, alpha)
        lmax, n_neg = stats.tolist()  # the path's single host sync
        if n_neg:
            raise RuntimeError(f"LengthRegulator: {n_neg} negative duration(s)")
        if lmax > INT32_MAX:
            raise RuntimeError(f"LengthRegulator: {lmax} frames in one utterance do not fit the int32 prefix sum")
        return gather(xs.contiguous(), cum, ilens_dev, int(lmax))
