"""Batched MelGAN vocoder on the library's kernels (DESIGN.md section 8).

The reference's default audio path is seungwonpark/melgan (`torch.hub.load("seungwonpark/melgan", "melgan")`,
inference.py:180-193): one eager call on one concatenated paragraph, and only with a network connection.  `MelGANVocoder`
runs the same generator batched and per utterance on libfs2b200.so (csrc/melgan.cu), loads that project's checkpoint
from a local file, and keeps the hub object's `inference(mel)` so that `vocoder.inference(mel)` works unchanged.

The module's parameters carry the checkpoint's 126 keys (`generator.1.{bias,weight_g,weight_v}` ... `generator.16.*`; the
list with shapes is tests/golden/melgan_state_dict_keys.json).  They are written from the published code, not checked
against a real checkpoint file.
"""
from __future__ import annotations

import ctypes as C
import os

import torch
import torch.nn as nn

from . import _lib

HOP = 256
N_MELS = 80
MAX_WAV_VALUE = 32768.0
_STAGES = ((512, 256, 8), (256, 128, 8), (128, 64, 2), (64, 32, 2))    # ConvTranspose1d (Cin, Cout, stride), k = 2 * stride


class _WNConv(nn.Module):
    """The parameters of one weight-normalised convolution, registered in `torch.nn.utils.weight_norm`'s order (bias,
    weight_g, weight_v).  weight = weight_g * weight_v / |weight_v|, the norm taken per index of dim 0: output channels of
    a Conv1d [Cout, Cin, k], *input* channels of a ConvTranspose1d [Cin, Cout, k]."""

    def __init__(self, cin: int, cout: int, k: int, transposed: bool = False):
        super().__init__()
        proto = nn.ConvTranspose1d(cin, cout, k) if transposed else nn.Conv1d(cin, cout, k)   # torch's default init
        v = proto.weight.detach()
        self.transposed = transposed
        self.bias = nn.Parameter(proto.bias.detach().clone())
        self.weight_g = nn.Parameter(torch.norm_except_dim(v, 2, 0).clone())
        self.weight_v = nn.Parameter(v.clone())

    def folded(self) -> torch.Tensor:
        """fp32 weight, computed on the CPU exactly as torch's weight_norm computes it there (`torch._weight_norm`)."""
        return torch._weight_norm(self.weight_v.detach().float().cpu(), self.weight_g.detach().float().cpu(), 0)


class _ResStack(nn.Module):
    def __init__(self, c: int):
        super().__init__()
        self.blocks = nn.ModuleList([nn.Sequential(nn.Identity(), nn.Identity(), _WNConv(c, c, 3), nn.Identity(), _WNConv(c, c, 1))
                                     for _ in range(3)])
        self.shortcuts = nn.ModuleList([_WNConv(c, c, 1) for _ in range(3)])


def _generator() -> nn.Sequential:
    """Parameter containers at the hub Generator's nn.Sequential indices (Identity where it has a parameter-free layer)."""
    mods = [nn.Identity(), _WNConv(N_MELS, 512, 7)]
    for cin, cout, s in _STAGES:
        mods += [nn.Identity(), _WNConv(cin, cout, 2 * s, transposed=True), _ResStack(cout)]
    mods += [nn.Identity(), nn.Identity(), _WNConv(32, 1, 7), nn.Identity()]
    return nn.Sequential(*mods)


class MelGANVocoder(nn.Module):
    """seungwonpark/melgan's `Generator(mel_channel=80)` on the H100 kernels.

    `forward(mels [B, Lmax, 80], olens [B])` -> (audio [B, Lmax * 256] fp32, alens = olens * 256).  Utterance b is the
    generator applied to mels[b, :olens[b]] followed by 10 frames of -11.5129, every reflection pad at its own edges,
    trimmed to olens[b] * 256 samples; it is bit-identical to a B = 1 call on its own frames whatever else is in the batch,
    audio past alens[b] is 0, and mel frames past olens[b] are never read.  `inference(mel [1, 80, T])` -> int16 [T * 256]
    is the hub object's method.  math_mode: "3xf16" (default, fp32-class), "f16", "tf32" or "fp32" for the GEMMs.  One
    host read per call (the device-side length and range checks)."""

    def __init__(self, math_mode: str = "3xf16"):
        super().__init__()
        if math_mode not in _lib.MATH_MODES:
            raise ValueError(f"math_mode must be one of {sorted(_lib.MATH_MODES)}")
        self.math_mode = math_mode
        self.mel_channel = N_MELS
        self.generator = _generator()
        self._layers = [m for m in self.modules() if isinstance(m, _WNConv)]      # state_dict order, 42 convolutions
        self._handles = {}       # device index -> (fs2_melgan_gen*, parameter fingerprint it was loaded from)
        self._ws = {}            # device index -> workspace tensor
        self._wws = {}           # device index -> window workspace tensor (fs2_melgan_window)
        self._epoch = 0

    def __del__(self):
        lib = _lib._lib
        for h, _ in getattr(self, "_handles", {}).values():
            if lib is not None and h:
                lib.fs2_melgan_destroy(h)

    # ---- checkpoints ----------------------------------------------------------------------------------------------
    @classmethod
    def from_checkpoint(cls, path_or_dict, math_mode: str = "3xf16") -> "MelGANVocoder":
        """seungwonpark/melgan's checkpoint (a dict with "model_g") or a bare generator state dict, given as a file path
        or as the loaded dict.  Either may hold `weight_g` / `weight_v` keys or plain `weight` keys (after
        `remove_weight_norm`, what the hub object holds); a plain weight w is stored as v = w, g = |w|, which folds back to
        w bit for bit.  A missing, unexpected or wrongly shaped key raises ValueError naming it."""
        sd = path_or_dict
        if isinstance(sd, (str, os.PathLike)):
            sd = torch.load(sd, map_location="cpu", weights_only=True)
        if not isinstance(sd, dict):
            raise ValueError("expected a checkpoint dict (with 'model_g') or a generator state dict")
        if "model_g" in sd:
            sd = sd["model_g"]
        voc = cls(math_mode=math_mode)
        voc.load_state_dict(voc._normalise(sd))
        return voc

    def _normalise(self, sd) -> dict:
        """Checkpoint dict -> this module's weight_g / weight_v state dict, validated key by key."""
        sd = dict(sd)
        prefixes = {name: m for name, m in self.named_modules() if isinstance(m, _WNConv)}
        out = {}
        for p, m in prefixes.items():
            if f"{p}.weight" in sd and (f"{p}.weight_g" in sd or f"{p}.weight_v" in sd):
                raise ValueError(f"unexpected key {p}.weight alongside {p}.weight_g / weight_v")
            wanted = [f"{p}.bias"] + ([f"{p}.weight"] if f"{p}.weight" in sd else [f"{p}.weight_g", f"{p}.weight_v"])
            for k in wanted:
                if k not in sd:
                    raise ValueError(f"missing key {k}")
            t = {k: sd.pop(k) for k in wanted}
            shapes = {f"{p}.bias": m.bias.shape, f"{p}.weight": m.weight_v.shape, f"{p}.weight_g": m.weight_g.shape,
                      f"{p}.weight_v": m.weight_v.shape}
            for k, v in t.items():
                if not torch.is_tensor(v) or tuple(v.shape) != tuple(shapes[k]):
                    got = tuple(v.shape) if torch.is_tensor(v) else type(v).__name__
                    raise ValueError(f"key {k} has shape {got}, expected {tuple(shapes[k])}")
            out[f"{p}.bias"] = t[f"{p}.bias"].float()
            if f"{p}.weight" in t:
                w = t[f"{p}.weight"].detach().float().cpu().contiguous()
                _, norms = torch._weight_norm_interface(w, torch.ones_like(m.weight_g, device="cpu"), 0)
                out[f"{p}.weight_g"] = norms.reshape(m.weight_g.shape)
                out[f"{p}.weight_v"] = w
            else:
                out[f"{p}.weight_g"] = t[f"{p}.weight_g"].float()
                out[f"{p}.weight_v"] = t[f"{p}.weight_v"].float()
        if sd:
            raise ValueError(f"unexpected key {sorted(sd)[0]}")
        return out

    def eval(self, inference: bool = False):
        """The hub object's signature.  inference=True removes weight norm there; here the folded weights are what the
        kernels use either way, so the audio is the same and the parameters keep their weight_g / weight_v form."""
        super().eval()
        return self

    def invalidate(self) -> None:
        """Force a weight reload on the next call (after in-place writes through `.data`, which torch does not version)."""
        self._epoch += 1

    # ---- device state ---------------------------------------------------------------------------------------------
    def _fingerprint(self):
        return (self._epoch,) + tuple((p.data_ptr(), p._version) for p in self.parameters())

    def _handle(self, device: torch.device):
        lib = _lib.load()
        key = self._fingerprint()
        ent = self._handles.get(device.index)
        if ent is not None and ent[1] == key:
            return ent[0]
        with torch.cuda.device(device):
            if ent is None:
                h = C.c_void_p()
                _lib.check(lib.fs2_melgan_create(C.byref(h), _lib.MATH_MODES[self.math_mode]), "fs2_melgan_create")
                h = h.value
            else:
                h = ent[0]
            ws = [m.folded().to(device).contiguous() for m in self._layers]
            bs = [m.bias.detach().float().to(device).contiguous() for m in self._layers]
            wp = (C.c_void_p * len(ws))(*[t.data_ptr() for t in ws])
            bp = (C.c_void_p * len(bs))(*[t.data_ptr() for t in bs])
            _lib.check(lib.fs2_melgan_load(h, wp, bp, _lib.stream_ptr(device)), "fs2_melgan_load")
        self._handles[device.index] = (h, key)
        return h

    def _workspace(self, h, B: int, L: int, device: torch.device) -> torch.Tensor:
        n = C.c_size_t()
        _lib.check(_lib.load().fs2_melgan_workspace_bytes(h, B, L, C.byref(n)), "fs2_melgan_workspace_bytes")
        ws = self._ws.get(device.index)
        if ws is None or ws.numel() < n.value:
            self._ws.pop(device.index, None)
            ws = torch.empty(n.value, dtype=torch.uint8, device=device)
            self._ws[device.index] = ws
        return ws

    def _inputs(self, mels, olens, check_size=None):
        if not torch.is_tensor(mels) or mels.dim() != 3 or mels.shape[2] != N_MELS or mels.shape[0] == 0 or mels.shape[1] == 0:
            raise ValueError(f"mels must be a non-empty [B, Lmax, {N_MELS}] tensor")
        if not torch.is_tensor(olens) or olens.dim() != 1 or olens.shape[0] != mels.shape[0]:
            raise ValueError(f"olens must be a [B={mels.shape[0]}] tensor")
        if olens.dtype.is_floating_point or olens.dtype == torch.bool:
            raise ValueError("olens must be an integer tensor")
        if not mels.is_cuda or not olens.is_cuda:
            raise ValueError("mels and olens must be CUDA tensors (the H100 path has no CPU fallback)")
        B, L, _ = mels.shape
        (check_size or self._check_size)(B, L)
        return mels.to(torch.float32).contiguous(), olens.to(device=mels.device, dtype=torch.int64).contiguous(), B, L

    def _check_size(self, B: int, L: int) -> None:
        """The limits fs2_melgan checks, raised here as ValueError: B * (Lmax + 10) * 256 sample rows below 2^31, and at
        most 65535 * 128 in fp32 mode (its CUDA-core GEMMs put 128-row tiles on grid.y)."""
        rows = B * (L + 10) * HOP
        if rows >= 1 << 31:
            raise ValueError(f"B * (Lmax + 10) * {HOP} must stay below 2^31 sample rows (B={B}, Lmax={L})")
        if self.math_mode == "fp32" and rows > 65535 * 128:
            raise ValueError(f"math_mode='fp32' takes at most 65535 * 128 sample rows, B * (Lmax + 10) * {HOP} = {rows} "
                             f"(B={B}, Lmax={L}); split the batch or use another math mode")

    def _window_workspace(self, h, B: int, n_frames: int, device: torch.device) -> torch.Tensor:
        n = C.c_size_t()
        _lib.check(_lib.load().fs2_melgan_window_workspace_bytes(h, B, n_frames, C.byref(n)), "fs2_melgan_window_workspace_bytes")
        ws = self._wws.get(device.index)
        if ws is None or ws.numel() < n.value:
            self._wws.pop(device.index, None)
            ws = torch.empty(n.value, dtype=torch.uint8, device=device)
            self._wws[device.index] = ws
        return ws

    @staticmethod
    def _check_frames(n_frames) -> None:
        if isinstance(n_frames, bool) or not isinstance(n_frames, int) or n_frames < 1:
            raise ValueError(f"n_frames / chunk_frames must be an int >= 1 (got {n_frames!r})")

    def _check_window_size(self, B: int, n_frames: int) -> None:
        """fs2_melgan_window's limits on the window's B * (256 * n_frames + 36) rows, raised here as ValueError."""
        self._check_frames(n_frames)
        rows = B * (n_frames * HOP + 36)
        if rows >= 1 << 31:
            raise ValueError(f"B * (256 * n_frames + 36) must stay below 2^31 window rows (B={B}, n_frames={n_frames})")
        if self.math_mode == "fp32" and rows > 65535 * 128:
            raise ValueError(f"math_mode='fp32' takes at most 65535 * 128 window rows, B * (256 * n_frames + 36) = {rows} "
                             f"(B={B}, n_frames={n_frames}); use fewer frames per window")

    def _starts(self, starts, B: int, device: torch.device) -> torch.Tensor:
        """starts as an int, a host list or tensor (checked >= 0 here) or a device tensor (checked on the device) -> [B]
        int64 on `device`."""
        if isinstance(starts, bool):
            raise ValueError("starts must be an int, a list or an integer tensor")
        if isinstance(starts, int):
            starts = [starts] * B
        if not torch.is_tensor(starts):
            try:
                starts = torch.tensor(starts)
            except (TypeError, ValueError, RuntimeError):
                raise ValueError("starts must be an int, a list or an integer tensor") from None
        if starts.dim() != 1 or starts.shape[0] != B:
            raise ValueError(f"starts must hold B={B} frame offsets")
        if starts.dtype.is_floating_point or starts.dtype == torch.bool or starts.is_complex():
            raise ValueError("starts must be an integer tensor")
        if not starts.is_cuda:
            if bool((starts < 0).any()):
                raise ValueError("every starts[b] must be >= 0")
        elif starts.device != device:
            raise ValueError("starts must be on the same device as mels")
        return starts.to(device=device, dtype=torch.int64).contiguous()

    def _window_call(self, h, mels, olens, starts, B: int, L: int, n_frames: int, audio: torch.Tensor, ld: int, status: torch.Tensor,
                     ws: torch.Tensor) -> None:
        dev = mels.device
        with torch.cuda.device(dev):
            _lib.check(_lib.load().fs2_melgan_window(h, _lib.ptr(mels), _lib.ptr(olens), _lib.ptr(starts), B, L, n_frames, audio.data_ptr(), ld,
                                                     _lib.ptr(status), _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev)), "fs2_melgan_window")

    def _check_status(self, status: torch.Tensor) -> None:
        s = int(status.item())                                                   # the call's one host read
        if s & _lib.FS2_MELGAN_BAD_LENGTH:
            raise ValueError("every olens[b] must lie in [1, Lmax]")
        if s & _lib.FS2_MELGAN_BAD_START:
            raise ValueError("every starts[b] must be >= 0")
        if s & _lib.FS2_MELGAN_RANGE:
            raise ValueError(f"activations exceed the range of the fp16 operand planes in math_mode={self.math_mode!r} "
                             f"(some GEMM input above {65504 / 16:g} in magnitude); use math_mode='fp32' or 'tf32'")

    # ---- synthesis ------------------------------------------------------------------------------------------------
    def forward(self, mels: torch.Tensor, olens: torch.Tensor, chunk_frames: int | None = None):
        """-> (audio [B, Lmax * 256] fp32, alens [B] int64 = olens * 256).

        chunk_frames=k: the same bits, computed as windows of k frames written straight into the output, with the
        workspace of one window (fs2_melgan_window): in fp32 mode this vocodes batches the whole call refuses.  Still one
        host read per call: the windows' status words are ORed on the device."""
        if chunk_frames is not None:
            return self._chunked(mels, olens, chunk_frames)
        mels, olens, B, L = self._inputs(mels, olens)
        dev = mels.device
        h = self._handle(dev)
        ws = self._workspace(h, B, L, dev)
        audio = torch.empty((B, L * HOP), dtype=torch.float32, device=dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.load().fs2_melgan(h, _lib.ptr(mels), _lib.ptr(olens), B, L, _lib.ptr(audio), _lib.ptr(status), _lib.ptr(ws),
                                              ws.numel(), _lib.stream_ptr(dev)), "fs2_melgan")
        self._check_status(status)
        return audio, olens * HOP

    def _window_inputs(self, mels, olens, n_frames):
        """_inputs with the window's limits in place of the whole call's (Lmax bounds only the per-utterance rows)."""
        self._check_frames(n_frames)
        def check(B, L):
            self._check_window_size(B, n_frames)
            if (L + 10) * HOP >= 1 << 31:
                raise ValueError(f"(Lmax + 10) * {HOP} must stay below 2^31 samples (Lmax={L})")
        return self._inputs(mels, olens, check)

    def window(self, mels: torch.Tensor, olens: torch.Tensor, starts, n_frames: int):
        """One window of the audio (DESIGN.md section 11): -> (audio [B, n_frames * 256] fp32, alens [B] int64 =
        clamp(olens - starts, 0, n_frames) * 256).  audio[b, :alens[b]] are samples [starts[b] * 256, ...) of
        `forward(mels, olens)[0][b]`, bit for bit; the rest is 0.  starts: an int (every utterance), a host list or tensor,
        or a device tensor.  Only mel frames [starts[b] - 6, starts[b] + n_frames + 6) below olens[b] are read; the
        workspace depends on B and n_frames only.  One host read per call."""
        mels, olens, B, L = self._window_inputs(mels, olens, n_frames)
        dev = mels.device
        starts = self._starts(starts, B, dev)
        h = self._handle(dev)
        ws = self._window_workspace(h, B, n_frames, dev)
        audio = torch.empty((B, n_frames * HOP), dtype=torch.float32, device=dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        self._window_call(h, mels, olens, starts, B, L, n_frames, audio, n_frames * HOP, status, ws)
        self._check_status(status)
        return audio, (olens - starts).clamp(0, n_frames) * HOP

    def stream(self, mels: torch.Tensor, olens: torch.Tensor, chunk_frames: int = 32):
        """Lockstep windows: yields (audio, alens) of `window(mels, olens, k * chunk_frames, chunk_frames)` for k = 0 ..
        ceil(Lmax / chunk_frames) - 1, the last one cut at Lmax, so that the chunks concatenated along time are
        `forward(mels, olens)`.  Utterances that have ended give rows of 0 (alens 0)."""
        self._check_frames(chunk_frames)
        L = mels.shape[1]
        for c0 in range(0, L, chunk_frames):
            yield self.window(mels, olens, c0, min(chunk_frames, L - c0))

    def _chunked(self, mels, olens, k: int):
        mels, olens, B, L = self._window_inputs(mels, olens, k)
        dev = mels.device
        h = self._handle(dev)
        ws = self._window_workspace(h, B, min(k, L), dev)
        audio = torch.empty((B, L * HOP), dtype=torch.float32, device=dev)
        c0s = list(range(0, L, k))
        starts = torch.tensor(c0s, dtype=torch.int64).repeat_interleave(B).reshape(len(c0s), B).to(dev)
        status = torch.empty((len(c0s),), dtype=torch.int32, device=dev)
        for i, c0 in enumerate(c0s):
            n = min(k, L - c0)
            self._window_call(h, mels, olens, starts[i], B, L, n, audio[:, c0 * HOP:], L * HOP, status[i: i + 1], ws)
        bits = torch.tensor([_lib.FS2_MELGAN_BAD_LENGTH, _lib.FS2_MELGAN_RANGE, _lib.FS2_MELGAN_BAD_START], dtype=torch.int32, device=dev)
        self._check_status(((status[:, None] & bits) != 0).any(0).int().mul(bits).sum().reshape(1))
        return audio, olens * HOP

    @staticmethod
    def quantize(audio: torch.Tensor) -> torch.Tensor:
        """The hub object's int16 conversion: * 32768, clamp to [-32768, 32767], truncate toward zero."""
        return (MAX_WAV_VALUE * audio).clamp(min=-MAX_WAV_VALUE, max=MAX_WAV_VALUE - 1).short()

    def inference(self, mel: torch.Tensor) -> torch.Tensor:
        """seungwonpark/melgan's `inference`: mel [1, 80, T] (or [80, T]) -> int16 audio [T * 256]."""
        if not torch.is_tensor(mel) or not (mel.dim() == 3 and mel.shape[0] == 1 or mel.dim() == 2) or mel.shape[-2] != N_MELS:
            raise ValueError(f"mel must be a [1, {N_MELS}, T] tensor")
        m = mel.reshape(1, N_MELS, -1).transpose(1, 2)
        olens = torch.full((1,), m.shape[1], dtype=torch.int64, device=m.device)
        audio, _ = self.forward(m, olens)
        return self.quantize(audio[0])
