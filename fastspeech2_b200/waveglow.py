"""Batched WaveGlow vocoder on the library's kernels (DESIGN.md section 9).

The reference's notebook reaches NVIDIA's WaveGlow through `torch.hub.load('nvidia/DeepLearningExamples:torchhub',
'nvidia_waveglow')` (demo_fastspeech2.ipynb, "Waveglow"): a network download, then one eager `infer` call on one
concatenated paragraph.  `WaveGlowVocoder` runs the same model batched and per utterance on libfs2b200.so
(csrc/waveglow.cu), loads DeepLearningExamples' checkpoint from a local file, and keeps the hub object's `infer(mel, sigma)`
and `remove_weightnorm(model)` so that the notebook's calls work unchanged.

The module's parameters carry the checkpoint's 938 keys (`upsample.*`, `WN.{k}.{start,in_layers.{i},cond_layers.{i},
res_skip_layers.{i}}.{bias,weight_g,weight_v}`, `WN.{k}.end.*`, `convinv.{k}.conv.weight`; the list with shapes at
n_channels = 512 is tests/golden/waveglow_state_dict_keys.json).  They are written from the published code, not checked
against a real checkpoint file.  n_channels C is read from the checkpoint's shapes: the published sizes are 256 and 512,
and which one NVIDIA's file uses is an assumption `from_checkpoint` checks rather than a fact this module relies on.
"""
from __future__ import annotations

import ctypes as C
import math
import os

import torch
import torch.nn as nn

from . import _lib
from .melgan import _WNConv

HOP = 256
N_MELS = 80
N_GROUP = 8
STEPS = HOP // N_GROUP              # step rows (groups of 8 samples) per mel frame
N_FLOWS, N_LAYERS = 12, 8
HALO = 96                           # frames a window's buffer holds on each side of its core: ceil(12 * 255 / 32)


def flow_channels(k: int) -> int:
    """Audio channels flow k works on: 8, 8, 8, 8, 6, 6, 6, 6, 4, 4, 4, 4."""
    return N_GROUP - 2 * (k // 4)


class _Conv(nn.Module):
    """A plain convolution's parameters (weight, bias), in nn.Conv1d's registration order."""

    def __init__(self, shape, n_bias: int = 0):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros(shape))
        if n_bias:
            self.bias = nn.Parameter(torch.zeros(n_bias))


class _Inv(nn.Module):
    """Invertible1x1Conv's parameter: conv.weight [c, c, 1], a random rotation as DeepLearningExamples initialises it."""

    def __init__(self, c: int):
        super().__init__()
        W = torch.linalg.qr(torch.randn(c, c))[0]
        if torch.det(W) < 0:
            W[:, 0] = -W[:, 0]
        self.conv = _Conv((c, c, 1))
        self.conv.weight.data.copy_(W[..., None])


class _WN(nn.Module):
    def __init__(self, n_half: int, c: int):
        super().__init__()
        self.in_layers = nn.ModuleList([_WNConv(c, 2 * c, 3) for _ in range(N_LAYERS)])
        self.res_skip_layers = nn.ModuleList([_WNConv(c, 2 * c if i < N_LAYERS - 1 else c, 1) for i in range(N_LAYERS)])
        self.cond_layers = nn.ModuleList([_WNConv(N_MELS * N_GROUP, 2 * c, 1) for _ in range(N_LAYERS)])
        self.start = _WNConv(n_half, c, 1)
        self.end = _Conv((2 * n_half, c, 1), 2 * n_half)           # zero-initialised, as in the published model


class WaveGlowVocoder(nn.Module):
    """DeepLearningExamples' `WaveGlow` (n_mel_channels 80, n_flows 12, n_group 8, n_early_every 4, n_early_size 2, WN 8
    layers of kernel 3, n_channels C) on the H100 kernels.

    `forward(mels [B, Lmax, 80], olens [B], *, sigma=1.0, seed=None, z=None)` -> (audio [B, Lmax * 256] fp32,
    alens = olens * 256).  Utterance b is `infer` on mels[b, :olens[b]] alone, every dilated convolution zero-padded at its
    own edges; it is bit-identical to a B = 1 call with the same noise whatever else is in the batch, audio past alens[b]
    is 0, and mel frames past olens[b] and z steps past olens[b] * 32 are never read.

    Noise: z [B, 8, Lmax * 32] in the layout `WaveGlow.forward` returns (channels 0-1 the early output of flow 4, 2-3 that
    of flow 8, 4-7 the last four), or drawn on the device per utterance from Philox4x32-10 keyed by a seed: `seed` an int
    s (utterance b gets s + b), a [B] integer tensor, or None (one int64 from torch's CPU generator, so consecutive calls
    differ and `torch.manual_seed` makes them reproducible).  `noise(olens, Lmax, seed)` returns the z a seeded call uses.
    The flows receive fp32(sigma * z).

    math_mode: "3xf16" (default, fp32-class), "f16", "tf32" or "fp32" for the GEMMs.  One host read per call (the
    device-side length and range checks).

    Streaming (DESIGN.md section 12): `window(mels, olens, starts, n_frames, seed=...)` computes n_frames frames of audio
    per utterance from starts[b], bit-identical to the same samples of `forward` with the same noise; `stream(...)` yields
    lockstep windows whose concatenation is `forward`, and `forward(..., chunk_frames=k)` computes the whole call's bits
    window by window.  A window's workspace depends on B and n_frames only."""

    def __init__(self, n_channels: int = 512, math_mode: str = "3xf16"):
        super().__init__()
        if math_mode not in _lib.MATH_MODES:
            raise ValueError(f"math_mode must be one of {sorted(_lib.MATH_MODES)}")
        if not isinstance(n_channels, int) or n_channels < 64 or n_channels > 1024 or n_channels % 64:
            raise ValueError(f"n_channels must be a multiple of 64 in [64, 1024] (the published models use 256 or 512), "
                             f"got {n_channels}")
        self.math_mode = math_mode
        self.n_channels = n_channels
        self.n_mel_channels, self.n_flows, self.n_group = N_MELS, N_FLOWS, N_GROUP
        self.upsample = _Conv((N_MELS, N_MELS, 1024), N_MELS)
        with torch.no_grad():                            # nn.ConvTranspose1d's default init
            nn.init.kaiming_uniform_(self.upsample.weight, a=math.sqrt(5))
            bound = 1 / math.sqrt(self.upsample.weight.shape[1] * 1024)
            self.upsample.bias.uniform_(-bound, bound)
        self.WN = nn.ModuleList([_WN(flow_channels(k) // 2, n_channels) for k in range(N_FLOWS)])
        self.convinv = nn.ModuleList([_Inv(flow_channels(k)) for k in range(N_FLOWS)])
        self._handles = {}       # device index -> (fs2_waveglow_net*, parameter fingerprint it was loaded from)
        self._ws = {}            # device index -> workspace tensor
        self._wws = {}           # device index -> window workspace tensor
        self._epoch = 0

    def __del__(self):
        lib = _lib._lib
        for h, _ in getattr(self, "_handles", {}).values():
            if lib is not None and h:
                lib.fs2_waveglow_destroy(h)

    # ---- checkpoints ----------------------------------------------------------------------------------------------
    @classmethod
    def from_checkpoint(cls, path_or_dict, math_mode: str = "3xf16") -> "WaveGlowVocoder":
        """DeepLearningExamples' checkpoint (a dict with "state_dict") or a bare state dict, given as a file path or as
        the loaded dict; keys may carry a leading "module." (a DistributedDataParallel save).  WN convolutions may hold
        `weight_g` / `weight_v` or plain `weight` keys (after `remove_weightnorm`); a plain weight w is stored as v = w,
        g = |w|, which folds back to w.  n_channels is read from WN.0.start's bias and checked against every other key: a
        missing, unexpected or wrongly shaped key raises ValueError naming it."""
        sd = path_or_dict
        if isinstance(sd, (str, os.PathLike)):
            sd = torch.load(sd, map_location="cpu", weights_only=True)
        if not isinstance(sd, dict):
            raise ValueError("expected a checkpoint dict (with 'state_dict') or a WaveGlow state dict")
        if "state_dict" in sd:
            sd = sd["state_dict"]
        if sd and all(isinstance(k, str) and k.startswith("module.") for k in sd):
            sd = {k[len("module."):]: v for k, v in sd.items()}
        b = sd.get("WN.0.start.bias")
        if not torch.is_tensor(b) or b.dim() != 1:
            raise ValueError("missing key WN.0.start.bias (n_channels is read from it)")
        voc = cls(n_channels=int(b.shape[0]), math_mode=math_mode)
        voc.load_state_dict(voc._normalise(sd))
        return voc

    def _normalise(self, sd) -> dict:
        """Checkpoint dict -> this module's state dict, validated key by key."""
        sd = dict(sd)
        out = {}
        wn = {name: m for name, m in self.named_modules() if isinstance(m, _WNConv)}
        for p, m in wn.items():
            if f"{p}.weight" in sd and (f"{p}.weight_g" in sd or f"{p}.weight_v" in sd):
                raise ValueError(f"unexpected key {p}.weight alongside {p}.weight_g / weight_v")
            wanted = [f"{p}.bias"] + ([f"{p}.weight"] if f"{p}.weight" in sd else [f"{p}.weight_g", f"{p}.weight_v"])
            shapes = {f"{p}.bias": m.bias.shape, f"{p}.weight": m.weight_v.shape, f"{p}.weight_g": m.weight_g.shape,
                      f"{p}.weight_v": m.weight_v.shape}
            t = self._take(sd, wanted, shapes)
            out[f"{p}.bias"] = t[f"{p}.bias"]
            if f"{p}.weight" in t:
                w = t[f"{p}.weight"].contiguous()
                _, norms = torch._weight_norm_interface(w, torch.ones_like(m.weight_g, device="cpu"), 0)
                out[f"{p}.weight_g"] = norms.reshape(m.weight_g.shape)
                out[f"{p}.weight_v"] = w
            else:
                out[f"{p}.weight_g"] = t[f"{p}.weight_g"]
                out[f"{p}.weight_v"] = t[f"{p}.weight_v"]
        own = self.state_dict()
        plain = [k for k in own if k not in out]
        out.update(self._take(sd, plain, {k: own[k].shape for k in plain}))
        if sd:
            raise ValueError(f"unexpected key {sorted(sd)[0]}")
        return out

    @staticmethod
    def _take(sd: dict, keys, shapes) -> dict:
        t = {}
        for k in keys:
            if k not in sd:
                raise ValueError(f"missing key {k}")
            v = sd.pop(k)
            if not torch.is_tensor(v) or tuple(v.shape) != tuple(shapes[k]):
                got = tuple(v.shape) if torch.is_tensor(v) else type(v).__name__
                raise ValueError(f"key {k} has shape {got}, expected {tuple(shapes[k])}")
            t[k] = v.detach().float().cpu()
        return t

    @staticmethod
    def remove_weightnorm(model):
        """The hub object's surface (`waveglow = waveglow.remove_weightnorm(waveglow)`).  The kernels run on the folded
        weights either way, so the parameters keep their weight_g / weight_v form and the audio is the same."""
        return model

    def invalidate(self) -> None:
        """Force a weight reload on the next call (after in-place writes through `.data`, which torch does not version)."""
        self._epoch += 1

    # ---- device state ---------------------------------------------------------------------------------------------
    def _fingerprint(self):
        return (self._epoch,) + tuple((p.data_ptr(), p._version) for p in self.parameters())

    def _tensors(self):
        """The 638 fp32 CPU tensors of fs2_waveglow_load, in its order (weight norm folded, W_inverse in float64)."""
        plain = lambda t: t.detach().float().cpu().contiguous()
        ts = [plain(self.upsample.weight), plain(self.upsample.bias)]
        for k in range(N_FLOWS):
            wn = self.WN[k]
            ts += [wn.start.folded(), plain(wn.start.bias)]
            for layers in (wn.in_layers, wn.cond_layers, wn.res_skip_layers):
                for m in layers:
                    ts += [m.folded(), plain(m.bias)]
            W = self.convinv[k].conv.weight.detach().cpu().double()[:, :, 0]
            ts += [plain(wn.end.weight), plain(wn.end.bias), torch.linalg.inv(W).float().contiguous()]
        return ts

    def _handle(self, device: torch.device):
        lib = _lib.load()
        key = self._fingerprint()
        ent = self._handles.get(device.index)
        if ent is not None and ent[1] == key:
            return ent[0]
        with torch.cuda.device(device):
            if ent is None:
                h = C.c_void_p()
                _lib.check(lib.fs2_waveglow_create(C.byref(h), _lib.MATH_MODES[self.math_mode], self.n_channels), "fs2_waveglow_create")
                h = h.value
            else:
                h = ent[0]
            ts = [t.to(device) for t in self._tensors()]
            tp = (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])
            _lib.check(lib.fs2_waveglow_load(h, tp, len(ts), _lib.stream_ptr(device)), "fs2_waveglow_load")
            torch.cuda.current_stream(device).synchronize()       # the staging tensors are freed on return
        self._handles[device.index] = (h, key)
        return h

    def _workspace(self, h, B: int, L: int, device: torch.device) -> torch.Tensor:
        n = C.c_size_t()
        _lib.check(_lib.load().fs2_waveglow_workspace_bytes(h, B, L, C.byref(n)), "fs2_waveglow_workspace_bytes")
        ws = self._ws.get(device.index)
        if ws is None or ws.numel() < n.value:
            self._ws.pop(device.index, None)
            ws = torch.empty(n.value, dtype=torch.uint8, device=device)
            self._ws[device.index] = ws
        return ws

    def _inputs(self, mels, olens, sigma, seed, z, check_size=None):
        """Validated (mels fp32, olens int64, B, Lmax, sigma, seeds or None, z fp32 or None); every check that needs no
        device runs before the one that asks for CUDA tensors.  check_size(B, Lmax): the limits (default: the whole
        call's)."""
        if not torch.is_tensor(mels) or mels.dim() != 3 or mels.shape[2] != N_MELS or mels.shape[0] == 0 or mels.shape[1] == 0:
            raise ValueError(f"mels must be a non-empty [B, Lmax, {N_MELS}] tensor")
        if not mels.dtype.is_floating_point:
            raise ValueError("mels must be a floating-point tensor")
        if not torch.is_tensor(olens) or olens.dim() != 1 or olens.shape[0] != mels.shape[0]:
            raise ValueError(f"olens must be a [B={mels.shape[0]}] tensor")
        if olens.dtype.is_floating_point or olens.dtype.is_complex or olens.dtype == torch.bool:
            raise ValueError("olens must be an integer tensor")
        B, L, _ = mels.shape
        sigma = self._sigma(sigma)
        seeds = None
        if z is not None:
            if seed is not None:
                raise ValueError("pass either z or seed, not both")
            if not torch.is_tensor(z) or tuple(z.shape) != (B, N_GROUP, L * STEPS) or not z.dtype.is_floating_point:
                raise ValueError(f"z must be a [B={B}, {N_GROUP}, Lmax * {STEPS} = {L * STEPS}] floating-point tensor")
        else:
            seeds = self._seeds(seed, B, mels.device)
        if not mels.is_cuda or not olens.is_cuda or (z is not None and z.device != mels.device):
            raise ValueError("mels, olens and z must be CUDA tensors on one device (the H100 path has no CPU fallback)")
        (check_size or self._check_size)(B, L)
        if z is not None:
            z = z.to(torch.float32).contiguous()
        return mels.to(torch.float32).contiguous(), olens.to(device=mels.device, dtype=torch.int64).contiguous(), B, L, sigma, seeds, z

    def _check_size(self, B: int, L: int) -> None:
        """The limits fs2_waveglow checks, raised here as ValueError: B * Lmax * 32 step rows below 2^31, and at most
        65535 * 128 in fp32 mode (its CUDA-core GEMMs put 128-row tiles on grid.y)."""
        rows = B * L * STEPS
        if rows >= 1 << 31:
            raise ValueError(f"B * Lmax * {STEPS} must stay below 2^31 step rows (B={B}, Lmax={L})")
        if self.math_mode == "fp32" and rows > 65535 * 128:
            raise ValueError(f"math_mode='fp32' takes at most 65535 * 128 step rows, B * Lmax * {STEPS} = {rows} "
                             f"(B={B}, Lmax={L}); split the batch or use another math mode")

    @staticmethod
    def _seeds(seed, B: int, device) -> torch.Tensor:
        if seed is None:
            seed = int(torch.randint(-2 ** 63, 2 ** 63 - 1, (), dtype=torch.int64))
        if isinstance(seed, bool) or not (isinstance(seed, int) or torch.is_tensor(seed)):
            raise ValueError("seed must be an int, a [B] integer tensor or None")
        if isinstance(seed, int):
            if not -2 ** 63 <= seed < 2 ** 63:
                raise ValueError("an int seed must fit in int64")
            return (torch.arange(B, dtype=torch.int64) + seed).to(device)      # wraps in int64
        if seed.dim() != 1 or seed.shape[0] != B or seed.dtype.is_floating_point or seed.dtype.is_complex or seed.dtype == torch.bool:
            raise ValueError(f"a seed tensor must be a [B={B}] integer tensor")
        return seed.to(device=device, dtype=torch.int64).contiguous()

    @staticmethod
    def _sigma(sigma) -> float:
        if isinstance(sigma, bool) or not isinstance(sigma, (int, float)) or not math.isfinite(sigma) or sigma < 0:
            raise ValueError(f"sigma must be a finite number >= 0, got {sigma!r}")
        return float(sigma)

    def _check_status(self, status: torch.Tensor) -> None:
        s = int(status.item())                                                   # the call's one host read
        if s & _lib.FS2_WAVEGLOW_BAD_LENGTH:
            raise ValueError("every olens[b] must lie in [1, Lmax]")
        if s & _lib.FS2_WAVEGLOW_BAD_START:
            raise ValueError("every starts[b] must be >= 0")
        if s & _lib.FS2_WAVEGLOW_RANGE:
            raise ValueError(f"activations exceed the range of the fp16 operand planes in math_mode={self.math_mode!r} "
                             f"(some GEMM input above {65504 / 16:g} in magnitude); use math_mode='fp32' or 'tf32'")

    # ---- synthesis ------------------------------------------------------------------------------------------------
    @classmethod
    def noise(cls, olens: torch.Tensor, Lmax: int, seed) -> torch.Tensor:
        """The standard-normal draw of a seeded call: z [B, 8, Lmax * 32] on olens' device, 0 at steps t >= olens[b] * 32."""
        if not torch.is_tensor(olens) or olens.dim() != 1 or olens.shape[0] == 0 or not olens.is_cuda:
            raise ValueError("olens must be a non-empty [B] CUDA tensor")
        if olens.dtype.is_floating_point or olens.dtype.is_complex or olens.dtype == torch.bool:
            raise ValueError("olens must be an integer tensor")
        if isinstance(Lmax, bool) or not isinstance(Lmax, int) or Lmax < 1 or olens.shape[0] * Lmax * STEPS >= 1 << 31:
            raise ValueError("Lmax must be a positive int with B * Lmax * 32 below 2^31")
        dev = olens.device
        B = olens.shape[0]
        seeds = cls._seeds(seed, B, dev)
        ol = olens.to(torch.int64).contiguous()
        z = torch.empty(B, N_GROUP, Lmax * STEPS, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.load().fs2_waveglow_noise(_lib.ptr(seeds), _lib.ptr(ol), B, Lmax, _lib.ptr(z), _lib.stream_ptr(dev)),
                       "fs2_waveglow_noise")
        return z

    def forward(self, mels: torch.Tensor, olens: torch.Tensor, *, sigma: float = 1.0, seed=None, z=None, chunk_frames: int | None = None):
        """-> (audio [B, Lmax * 256] fp32, alens [B] int64 = olens * 256).

        chunk_frames=k: the same bits, computed as windows of k frames written straight into the output, with the
        workspace of one window (fs2_waveglow_window): in fp32 mode this vocodes batches the whole call refuses.  seed=None
        draws the same one int64 as the whole call.  Still one host read per call: the windows' status words are ORed on
        the device."""
        if chunk_frames is not None:
            return self._chunked(mels, olens, chunk_frames, sigma, seed, z)
        mels, olens, B, L, sigma, seeds, z = self._inputs(mels, olens, sigma, seed, z)
        dev = mels.device
        h = self._handle(dev)
        ws = self._workspace(h, B, L, dev)
        audio = torch.empty((B, L * HOP), dtype=torch.float32, device=dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.load().fs2_waveglow(h, _lib.ptr(mels), _lib.ptr(olens), B, L, sigma, _lib.ptr(seeds), _lib.ptr(z),
                                                _lib.ptr(audio), _lib.ptr(status), _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev)),
                       "fs2_waveglow")
        self._check_status(status)
        return audio, olens * HOP

    # ---- windows (DESIGN.md section 12) ----------------------------------------------------------------------------
    @staticmethod
    def _check_frames(n_frames) -> None:
        if isinstance(n_frames, bool) or not isinstance(n_frames, int) or n_frames < 1:
            raise ValueError(f"n_frames / chunk_frames must be an int >= 1 (got {n_frames!r})")

    def _check_window_size(self, B: int, n_frames: int) -> None:
        """fs2_waveglow_window's limits on the window's B * (n_frames + 192) * 32 step rows, raised here as ValueError."""
        self._check_frames(n_frames)
        rows = B * (n_frames + 2 * HALO) * STEPS
        if rows >= 1 << 31:
            raise ValueError(f"B * (n_frames + {2 * HALO}) * {STEPS} must stay below 2^31 window rows (B={B}, n_frames={n_frames})")
        if self.math_mode == "fp32" and rows > 65535 * 128:
            raise ValueError(f"math_mode='fp32' takes at most 65535 * 128 window rows, B * (n_frames + {2 * HALO}) * {STEPS} = {rows} "
                             f"(B={B}, n_frames={n_frames}); use fewer frames per window")

    def _window_inputs(self, mels, olens, n_frames, sigma, seed, z):
        """_inputs with the window's limits in place of the whole call's (Lmax bounds only z's and mels' layout)."""
        self._check_frames(n_frames)

        def check(B, L):
            self._check_window_size(B, n_frames)
            if L * STEPS >= 1 << 31:
                raise ValueError(f"Lmax * {STEPS} must stay below 2^31 steps (Lmax={L})")
        return self._inputs(mels, olens, sigma, seed, z, check)

    def _window_workspace(self, h, B: int, n_frames: int, device: torch.device) -> torch.Tensor:
        n = C.c_size_t()
        _lib.check(_lib.load().fs2_waveglow_window_workspace_bytes(h, B, n_frames, C.byref(n)), "fs2_waveglow_window_workspace_bytes")
        ws = self._wws.get(device.index)
        if ws is None or ws.numel() < n.value:
            self._wws.pop(device.index, None)
            ws = torch.empty(n.value, dtype=torch.uint8, device=device)
            self._wws[device.index] = ws
        return ws

    @staticmethod
    def _starts(starts, B: int, device: torch.device) -> torch.Tensor:
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

    def _window_call(self, h, mels, olens, starts, B: int, L: int, n_frames: int, sigma: float, seeds, z, audio: torch.Tensor, ld: int,
                     status: torch.Tensor, ws: torch.Tensor) -> None:
        dev = mels.device
        with torch.cuda.device(dev):
            _lib.check(_lib.load().fs2_waveglow_window(h, _lib.ptr(mels), _lib.ptr(olens), _lib.ptr(starts), B, L, n_frames, sigma,
                                                       _lib.ptr(seeds), _lib.ptr(z), audio.data_ptr(), ld, _lib.ptr(status), _lib.ptr(ws),
                                                       ws.numel(), _lib.stream_ptr(dev)), "fs2_waveglow_window")

    def window(self, mels: torch.Tensor, olens: torch.Tensor, starts, n_frames: int, *, sigma: float = 1.0, seed=None, z=None):
        """One window of the audio (DESIGN.md section 12): -> (audio [B, n_frames * 256] fp32, alens [B] int64 =
        clamp(olens - starts, 0, n_frames) * 256).  audio[b, :alens[b]] are samples [starts[b] * 256, ...) of
        `forward(mels, olens, sigma=sigma, seed=seed / z=z)[0][b]`, bit for bit; the rest is 0.  starts: an int (every
        utterance), a host list or tensor, or a device tensor.  The noise must be given (seed or z [B, 8, Lmax * 32]): a
        window is only meaningful against a whole call with the same draw.  Only mel frames [starts[b] - 99, starts[b] +
        n_frames + 96) below olens[b] and the z steps 32 times those frames are read; the workspace depends on B and
        n_frames only.  One host read per call."""
        if seed is None and z is None:
            raise ValueError("window needs the noise: pass seed (an int or a [B] tensor) or z, as the whole call it continues")
        mels, olens, B, L, sigma, seeds, z = self._window_inputs(mels, olens, n_frames, sigma, seed, z)
        dev = mels.device
        starts = self._starts(starts, B, dev)
        h = self._handle(dev)
        ws = self._window_workspace(h, B, n_frames, dev)
        audio = torch.empty((B, n_frames * HOP), dtype=torch.float32, device=dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        self._window_call(h, mels, olens, starts, B, L, n_frames, sigma, seeds, z, audio, n_frames * HOP, status, ws)
        self._check_status(status)
        return audio, (olens - starts).clamp(0, n_frames) * HOP

    @staticmethod
    def _resolve_seed(seed, z):
        """seed=None without z: the one int64 the whole call would draw, drawn once for every window of a stream."""
        if seed is None and z is None:
            return int(torch.randint(-2 ** 63, 2 ** 63 - 1, (), dtype=torch.int64))
        return seed

    def stream(self, mels: torch.Tensor, olens: torch.Tensor, chunk_frames: int = 32, *, sigma: float = 1.0, seed=None, z=None):
        """Lockstep windows: yields (audio, alens) of `window(mels, olens, k * chunk_frames, chunk_frames, ...)` for k = 0 ..
        ceil(Lmax / chunk_frames) - 1, the last one cut at Lmax, so that the chunks concatenated along time are
        `forward(mels, olens, sigma=sigma, seed=seed, z=z)`; seed=None draws the whole call's one int64, once.  Utterances
        that have ended give rows of 0 (alens 0)."""
        self._check_frames(chunk_frames)
        seed = self._resolve_seed(seed, z)
        if torch.is_tensor(mels) and mels.dim() == 3 and seed is not None:
            seed = self._seeds(seed, mels.shape[0], mels.device)          # validated and moved once
        L = mels.shape[1]
        for c0 in range(0, L, chunk_frames):
            yield self.window(mels, olens, c0, min(chunk_frames, L - c0), sigma=sigma, seed=seed, z=z)

    def _chunked(self, mels, olens, k: int, sigma, seed, z):
        self._check_frames(k)
        seed = self._resolve_seed(seed, z)
        mels, olens, B, L, sigma, seeds, z = self._window_inputs(mels, olens, k, sigma, seed, z)
        dev = mels.device
        h = self._handle(dev)
        ws = self._window_workspace(h, B, min(k, L), dev)
        audio = torch.empty((B, L * HOP), dtype=torch.float32, device=dev)
        c0s = list(range(0, L, k))
        starts = torch.tensor(c0s, dtype=torch.int64).repeat_interleave(B).reshape(len(c0s), B).to(dev)
        status = torch.empty((len(c0s),), dtype=torch.int32, device=dev)
        for i, c0 in enumerate(c0s):
            n = min(k, L - c0)
            self._window_call(h, mels, olens, starts[i], B, L, n, sigma, seeds, z, audio[:, c0 * HOP:], L * HOP, status[i: i + 1], ws)
        bits = torch.tensor([_lib.FS2_WAVEGLOW_BAD_LENGTH, _lib.FS2_WAVEGLOW_RANGE, _lib.FS2_WAVEGLOW_BAD_START], dtype=torch.int32,
                            device=dev)
        self._check_status(((status[:, None] & bits) != 0).any(0).int().mul(bits).sum().reshape(1))
        return audio, olens * HOP

    def infer(self, spect: torch.Tensor, sigma: float = 1.0) -> torch.Tensor:
        """DeepLearningExamples' `infer`: spect [B, 80, T] -> audio [B, T * 256] fp32, fresh noise per call."""
        if not torch.is_tensor(spect) or spect.dim() != 3 or spect.shape[1] != N_MELS or spect.shape[0] == 0 or spect.shape[2] == 0:
            raise ValueError(f"spect must be a non-empty [B, {N_MELS}, T] tensor")
        m = spect.transpose(1, 2)
        olens = torch.full((m.shape[0],), m.shape[1], dtype=torch.int64, device=m.device)
        audio, _ = self.forward(m, olens, sigma=sigma)
        return audio
