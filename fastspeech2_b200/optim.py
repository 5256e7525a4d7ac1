"""The reference's optimizer (core/optimizer.py: NoamOpt over Adam(betas=(0.9, 0.98), eps=1e-9)) on the library's kernels.

    opt = get_std_opt(model, d_model, warmup, factor)     # same signature and surface as the reference's
    ...
    loss.backward()
    norm = opt.clip_and_step(grad_clip)                   # clip_grad_norm_ + NaN guard + NoamOpt.step(), no host sync
    opt.zero_grad()

`step()` is NoamOpt.step(): the counter advances, lr = rate(step), one Adam update, bit-identical to torch's foreach Adam
on the same gradients.  `clip_and_step(max_norm)` adds the deterministic gradient norm (fp64 chunk sums, fixed-order
reduction), the clip coefficient min(max_norm / (norm + 1e-6), 1) and the reference loop's NaN guard, all on the device:
it returns the norm as a 0-d CUDA tensor, and when the norm is NaN nothing changes (parameters, Adam state and the step
counter), which is what the reference loop's `continue` does.  The scaled gradients are not written back into `.grad`.
DESIGN.md section 15 has the arithmetic and the measurements."""
from __future__ import annotations

import ctypes as C
from typing import Iterable

import torch

from . import _lib

BETAS, EPS = (0.9, 0.98), 1e-9
_ENTRY_WORDS = 7            # fs2_optim_entry: param, grad, exp_avg, exp_avg_sq, step, numel, chunk0


def _require_cuda(params: list) -> None:
    dev = params[0].device if isinstance(params[0], torch.Tensor) else None
    for p in params:
        if not isinstance(p, torch.Tensor) or not p.is_cuda or p.dtype != torch.float32 or p.is_sparse or not p.is_contiguous():
            raise ValueError("NoamAdam: parameters must be contiguous dense CUDA float32 tensors")
        if p.device != dev:
            raise ValueError("NoamAdam: parameters must share one device")


class NoamAdam:
    """NoamOpt(model_size, factor, warmup, Adam(params, lr=0, betas=(0.9, 0.98), eps=1e-9)) with the update on the library's
    kernels.  The surface is NoamOpt's: step, zero_grad, rate, param_groups, _step, _rate, state_dict, load_state_dict;
    `optimizer` is a torch Adam that holds param_groups and state (exp_avg, exp_avg_sq, step) for state_dict purposes and
    is never stepped.  The step counter lives on the device; reading `_step` or `_rate` synchronises."""

    def __init__(self, params: Iterable[torch.Tensor], model_size, factor, warmup):
        params = list(params)
        if params and isinstance(params[0], dict):
            raise ValueError("NoamAdam: parameter groups are not supported; pass the parameters")
        if not params or not any(getattr(p, "requires_grad", False) for p in params):
            raise ValueError("NoamAdam: the model has no trainable parameters")
        _require_cuda(params)
        self.optimizer = torch.optim.Adam(params, lr=0, betas=BETAS, eps=EPS)
        self.params = params
        self.device = params[0].device
        self.warmup, self.factor, self.model_size = warmup, factor, model_size
        self._noam = torch.zeros(1, dtype=torch.int64, device=self.device)     # NoamOpt._step
        self._lr = torch.zeros(1, dtype=torch.float64, device=self.device)     # lr of the last step that ran
        self._steps = torch.zeros(len(params), dtype=torch.float32, device=self.device)   # torch Adam's state['step']
        self._key = None
        self._table = None
        self._numel = None
        self._ws = None
        self._updated: list = []

    # ---- NoamOpt surface ------------------------------------------------------------------------------------------------
    @property
    def param_groups(self):
        "the Adam groups, with lr set to _rate as NoamOpt.step() leaves it (synchronises)"
        rate = self._rate
        for g in self.optimizer.param_groups:
            g["lr"] = rate
        return self.optimizer.param_groups

    @property
    def _step(self) -> int:
        return int(self._noam.item())

    @_step.setter
    def _step(self, value) -> None:
        self._noam.fill_(int(value))

    @property
    def _rate(self) -> float:
        step = self._step
        return self.rate(step) if step > 0 else 0

    @_rate.setter
    def _rate(self, value) -> None:       # load_state_dict sets it; it is always rate(_step) of the same schedule
        pass

    def rate(self, step=None):
        "NoamOpt.rate, evaluated on the host exactly as the reference writes it"
        if step is None:
            step = self._step
        return self.factor * self.model_size ** (-0.5) * min(step ** (-0.5), step * self.warmup ** (-1.5))

    def zero_grad(self, set_to_none: bool = True) -> None:
        self.optimizer.zero_grad(set_to_none=set_to_none)

    def step(self) -> None:
        "NoamOpt.step(): counter + 1, lr = rate(counter), one Adam update on the current gradients (no clip)"
        args = self._prepare()
        if args is None:
            return
        _lib.check(_lib.load().fs2_optim_noam_adam(*args[:4], self._noam.data_ptr(), self._lr.data_ptr(), *args[4:]),
                   "fs2_optim_noam_adam")
        self._bump()

    def clip_and_step(self, max_norm: float) -> torch.Tensor:
        """clip_grad_norm_(params, max_norm) + the reference loop's NaN guard + step(), with no host synchronisation.
        Returns the total gradient norm (0-d fp32 CUDA tensor).  NaN norm: nothing is updated and the counter stays.
        The gradients are scaled inside the update; `.grad` keeps the unscaled values."""
        norm = torch.full((), float("nan"), dtype=torch.float32, device=self.device)
        args = self._prepare()
        if args is None:
            return norm
        _lib.check(_lib.load().fs2_optim_clip_noam_adam(*args[:4], float(max_norm), self._noam.data_ptr(), self._lr.data_ptr(),
                                                        norm.data_ptr(), *args[4:]), "fs2_optim_clip_noam_adam")
        self._bump()
        return norm

    def state_dict(self) -> dict:
        self._sync_steps_to_state()
        self.param_groups                 # lr = _rate in every group, as NoamOpt leaves it
        return {"_step": self._step, "warmup": self.warmup, "factor": self.factor, "model_size": self.model_size,
                "_rate": self._rate, "optimizer": self.optimizer.state_dict()}

    def load_state_dict(self, state_dict: dict) -> None:
        for key, value in state_dict.items():
            if key == "optimizer":
                self.optimizer.load_state_dict(value)
                self._sync_steps_from_state()
            else:
                setattr(self, key, value)

    # ---- internals --------------------------------------------------------------------------------------------------------
    def _hp(self) -> _lib.NoamAdamHp:
        g = self.optimizer.param_groups[0]
        (b1, b2), eps = g["betas"], g["eps"]
        return _lib.NoamAdamHp(self.factor * self.model_size ** (-0.5), self.warmup ** (-1.5), b1, b2, eps)

    def _state_of(self, i: int, p: torch.Tensor) -> dict:
        st = self.optimizer.state[p]
        if not st:                        # torch's lazy init at a parameter's first step
            st["step"] = torch.tensor(0.0, dtype=torch.float32)
            st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        return st

    def _prepare(self):
        """The entry table of the parameters that have a gradient; uploaded (from pinned memory, asynchronously) only when a
        pointer or the set of gradients changed.  Returns the library's leading and trailing arguments, or None."""
        rows, key = [], []
        for i, p in enumerate(self.params):
            g = p.grad
            if g is None:
                continue
            st = self._state_of(i, p)
            m, v = st["exp_avg"], st["exp_avg_sq"]
            k = (i, p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr())
            key.append(k)
            rows.append((i, p, g, m, v))
        if not rows:
            self._updated = []
            return None
        key = tuple(key)
        if key != self._key:
            self._upload(rows)
            self._key = key
        ws = self._ws
        self._hp_c = self._hp()
        return (self._table.data_ptr(), self._numel, len(rows), C.byref(self._hp_c), ws.data_ptr(), ws.numel(),
                _lib.stream_ptr(self.device))

    def _upload(self, rows) -> None:
        for i, p, g, m, v in rows:
            if not (g.is_cuda and g.device == self.device and g.dtype == torch.float32 and g.is_contiguous() and not g.is_sparse
                    and g.shape == p.shape):
                raise ValueError("NoamAdam: gradients must be contiguous dense CUDA float32 tensors shaped like their parameter")
            for t in (m, v):
                if not (t.device == self.device and t.dtype == torch.float32 and t.is_contiguous() and t.shape == p.shape):
                    raise ValueError("NoamAdam: Adam state must be contiguous CUDA float32 tensors shaped like the parameter")
        host = torch.empty(len(rows), _ENTRY_WORDS, dtype=torch.int64, pin_memory=True)
        chunk, base = 0, self._steps.data_ptr()
        numel = []
        for r, (i, p, g, m, v) in enumerate(rows):
            n = p.numel()
            host[r] = torch.tensor([p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), base + 4 * i, n, chunk])
            chunk += (n + _lib.FS2_OPTIM_CHUNK - 1) // _lib.FS2_OPTIM_CHUNK
            numel.append(n)
        if self._table is None or self._table.shape[0] < len(rows):
            self._table = torch.empty(len(self.params), _ENTRY_WORDS, dtype=torch.int64, device=self.device)
        self._table[:len(rows)].copy_(host, non_blocking=True)
        self._numel = (C.c_int64 * len(numel))(*numel)
        need = C.c_size_t(0)
        _lib.check(_lib.load().fs2_optim_ws_bytes(self._numel, len(numel), C.byref(need)), "fs2_optim_ws_bytes")
        if self._ws is None or self._ws.numel() < need.value:
            self._ws = torch.empty(need.value, dtype=torch.uint8, device=self.device)
        self._updated = [p for _, p, _, _, _ in rows]

    def _bump(self) -> None:
        # the kernels wrote the parameters through raw pointers: bump their version counters so that version-keyed caches
        # (the model's eval weight arena) see the update
        torch.autograd.graph.increment_version(self._updated)

    def _sync_steps_to_state(self) -> None:
        steps = self._steps.cpu()
        for i, p in enumerate(self.params):
            st = self.optimizer.state.get(p)
            if st:
                st["step"] = steps[i].clone()

    def _sync_steps_from_state(self) -> None:
        steps = torch.zeros(len(self.params), dtype=torch.float32)
        for i, p in enumerate(self.params):
            st = self.optimizer.state.get(p)
            if st and "step" in st:
                steps[i] = float(st["step"])
        self._steps.copy_(steps)
        self._key = None                  # the state tensors were replaced


def get_std_opt(model, d_model, warmup, factor) -> NoamAdam:
    "core/optimizer.py::get_std_opt on the library's kernels"
    return NoamAdam(model.parameters(), d_model, factor, warmup)
