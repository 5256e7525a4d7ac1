"""Host-side layer the signal modules share (MelGAN, HiFi-GAN, WaveGlow, Griffin-Lim, feature extraction): the per-device
handle and workspace caches, the status-word check, checkpoint reading and weight-norm normalisation, and the call surface
of the three neural vocoders: input and size checks, the whole call, and the windows (DESIGN.md sections 11, 12 and
17)."""
from __future__ import annotations

import ctypes as C
import itertools
import operator
import os

import torch
import torch.nn as nn

from . import _lib

HOP = 256                        # audio samples per mel frame
N_MELS = 80
MAX_WAV_VALUE = 32768.0


class Handles:
    """One library handle per device with the key it was loaded from; a call with another key reloads it in place."""

    def __init__(self, destroy: str):
        self._destroy = destroy  # the C entry that frees a handle
        self._ents = {}          # device index -> (handle, key)

    def get(self, device: torch.device, key, create, load):
        """The handle of `device`: create() -> handle on first use, then load(handle, device) whenever key changes."""
        ent = self._ents.get(device.index)
        if ent is not None and ent[1] == key:
            return ent[0]
        with torch.cuda.device(device):
            h = ent[0] if ent is not None else create()
            load(h, device)
        self._ents[device.index] = (h, key)
        return h

    def destroy_all(self) -> None:
        lib = _lib._lib
        for h, _ in self._ents.values():
            if lib is not None and h:
                getattr(lib, self._destroy)(h)


def query_bytes(entry: str, *args) -> int:
    """What a `*_workspace_bytes(..., size_t* bytes)` C entry answers for args."""
    n = C.c_size_t()
    _lib.check(getattr(_lib.load(), entry)(*args, C.byref(n)), entry)
    return n.value


def workspace(cache: dict, device: torch.device, nbytes: int) -> torch.Tensor:
    """cache[device.index]: a uint8 buffer of at least nbytes on `device`, grown on demand.  The smaller buffer goes back
    to the allocator before the larger one is taken, so growing never holds both."""
    ws = cache.get(device.index)
    if ws is not None and ws.numel() >= nbytes:
        return ws
    cache.pop(device.index, None)
    del ws
    ws = cache[device.index] = torch.empty(nbytes, dtype=torch.uint8, device=device)
    return ws


def check_status(status: torch.Tensor, table) -> None:
    """Raises ValueError(message) for the first (bit, message) of table whose bit is set in the device status word."""
    s = int(status.item())                                                   # the call's one host read
    for bit, message in table:
        if s & bit:
            raise ValueError(message)


# ---- checkpoints --------------------------------------------------------------------------------------------------

def read_checkpoint(path_or_dict, wrapper_key: str, what: str) -> dict:
    """A checkpoint given as a file path or as the loaded dict -> its state dict: what is under wrapper_key when the
    dict has that key, else the dict itself.  `what` names the bare state dict in the error."""
    sd = path_or_dict
    if isinstance(sd, (str, os.PathLike)):
        sd = torch.load(sd, map_location="cpu", weights_only=True)
    if not isinstance(sd, dict):
        raise ValueError(f"expected a checkpoint dict (with '{wrapper_key}') or {what}")
    return sd[wrapper_key] if wrapper_key in sd else sd



class _WNConv(nn.Module):
    """The parameters of one weight-normalised convolution, registered in `torch.nn.utils.weight_norm`'s order (bias,
    unless bias=False, weight_g, weight_v).  weight = weight_g * weight_v / |weight_v|, the norm taken per index of dim 0: output channels of
    a Conv1d [Cout, Cin, k], *input* channels of a ConvTranspose1d [Cin, Cout, k]."""

    def __init__(self, cin: int, cout: int, k: int, transposed: bool = False, bias: bool = True):
        super().__init__()
        proto = nn.ConvTranspose1d(cin, cout, k) if transposed else nn.Conv1d(cin, cout, k)   # torch's default init
        v = proto.weight.detach()
        self.transposed = transposed
        self.bias = nn.Parameter(proto.bias.detach().clone()) if bias else None
        self.weight_g = nn.Parameter(torch.norm_except_dim(v, 2, 0).clone())
        self.weight_v = nn.Parameter(v.clone())

    def folded(self) -> torch.Tensor:
        """fp32 weight, computed on the CPU exactly as torch's weight_norm computes it there (`torch._weight_norm`)."""
        return torch._weight_norm(self.weight_v.detach().float().cpu(), self.weight_g.detach().float().cpu(), 0)


def _take(sd: dict, keys, shapes) -> dict:
    """Pops keys from sd as fp32 CPU tensors: a missing key, then a wrongly shaped one, raises ValueError naming it."""
    for k in keys:
        if k not in sd:
            raise ValueError(f"missing key {k}")
    t = {}
    for k in keys:
        v = sd.pop(k)
        if not torch.is_tensor(v) or tuple(v.shape) != tuple(shapes[k]):
            got = tuple(v.shape) if torch.is_tensor(v) else type(v).__name__
            raise ValueError(f"key {k} has shape {got}, expected {tuple(shapes[k])}")
        t[k] = v.detach().float().cpu()
    return t


def normalise_checkpoint(module: nn.Module, sd) -> dict:
    """Checkpoint dict -> module's state dict, validated key by key.  A weight-normalised convolution (_WNConv) takes
    `weight_g` / `weight_v` keys or a plain `weight` (after `remove_weight_norm`), stored as v = w, g = |w|, which folds
    back to w bit for bit; every other key of the state dict is taken as it is.  A missing, unexpected or wrongly shaped
    key raises ValueError naming it."""
    sd = dict(sd)
    out = {}
    for p, m in module.named_modules():
        if not isinstance(m, _WNConv):
            continue
        if f"{p}.weight" in sd and (f"{p}.weight_g" in sd or f"{p}.weight_v" in sd):
            raise ValueError(f"unexpected key {p}.weight alongside {p}.weight_g / weight_v")
        wanted = [f"{p}.weight"] if f"{p}.weight" in sd else [f"{p}.weight_g", f"{p}.weight_v"]
        wanted = ([f"{p}.bias"] if m.bias is not None else []) + wanted
        shapes = {f"{p}.weight": m.weight_v.shape, f"{p}.weight_g": m.weight_g.shape, f"{p}.weight_v": m.weight_v.shape}
        if m.bias is not None:
            shapes[f"{p}.bias"] = m.bias.shape
        t = _take(sd, wanted, shapes)
        if m.bias is not None:
            out[f"{p}.bias"] = t[f"{p}.bias"]
        if f"{p}.weight" in t:
            w = t[f"{p}.weight"].contiguous()
            _, norms = torch._weight_norm_interface(w, torch.ones_like(m.weight_g, device="cpu"), 0)
            out[f"{p}.weight_g"] = norms.reshape(m.weight_g.shape)
            out[f"{p}.weight_v"] = w
        else:
            out[f"{p}.weight_g"] = t[f"{p}.weight_g"]
            out[f"{p}.weight_v"] = t[f"{p}.weight_v"]
    own = module.state_dict()
    for k in own:
        if k not in out:
            out.update(_take(sd, [k], {k: own[k].shape}))
    if sd:
        raise ValueError(f"unexpected key {sorted(sd)[0]}")
    return out


# ---- the neural vocoders --------------------------------------------------------------------------------------------

def ups_window_plan(rates, R: int, margin0: int, post: int = 3) -> dict:
    """The window plan of an upsampling chain (MelGAN, HiFi-GAN; DESIGN.md section 11; csrc/vocoder_window.cuh), walking
    back from the audio: the last convolution reads `post` rows on each side, each residual stack R, upsampling s (a
    polyphase ConvTranspose1d of k = 2 u_s) reads reach[s] input rows around its core, and level 0 holds margin0 rows more
    (the rows the first convolution leaves wrong at a window side that is not an utterance edge).  -> {"reach": [r_s],
    "halo": [h_s] (rows of level s on each side of its core; h_0 = r_0 + margin0, h_{s+1} = u_s r_s), "R": R}."""
    reach, halo, need = [0] * len(rates), [0] * (len(rates) + 1), post
    for s in reversed(range(len(rates))):
        need += R
        u = rates[s]
        t, p = divmod(-need, u)                          # output row -need = u t + p reads t - 1 (p < u / 2) or t
        reach[s] = need = -(t - 1 if p < u // 2 else t)
        halo[s + 1] = u * need
    halo[0] = need + margin0
    return {"reach": reach, "halo": halo, "R": R}


class NeuralVocoder(nn.Module):
    """What MelGANVocoder, HiFiGANVocoder and WaveGlowVocoder share around their C entries: the math mode; the handle,
    reloaded when a parameter changes; the mels / olens and size checks; the whole call with its workspace and status
    check; and the window layer (`window`'s inputs, `stream`'s loop, `forward(chunk_frames=)`).

    A subclass names its C entries by their prefix (_NAME: fs2_<_NAME>, fs2_<_NAME>_window, fs2_<_NAME>_destroy, the
    two *_workspace_bytes and the FS2_<_NAME> status bits) and the frames each utterance runs past olens (_TAIL), and
    provides _create() -> handle, _load(handle, device) and _rows(B, Lmax) -> (rows, their formula, their noun).  A whole
    call is call(h, mels, olens, B, Lmax, audio, status, ws), a window call call(h, mels, olens, starts, B, Lmax, n_frames,
    audio, audio_ld, status, ws).

    MelGAN, HiFi-GAN and BigVGAN, upsampling chains, also provide _chain() -> (upsample rates, stack reach R, level-0
    margin[, the last layer's reach when it is not 3]) and
    take the rest from here: _call and _window_call on their C entries, the window's rows from the chain's plan, and
    forward, window and stream.  WaveGlow, whose calls carry the noise, has its own calls, window rows and those three."""

    HOP = HOP
    _TAIL = 0

    def __init__(self, math_mode: str):
        super().__init__()
        if math_mode not in _lib.MATH_MODES:
            raise ValueError(f"math_mode must be one of {sorted(_lib.MATH_MODES)}")
        self.math_mode = math_mode
        self._handles = Handles(f"fs2_{self._NAME}_destroy")
        self._ws = {}            # device index -> workspace tensor
        self._wws = {}           # device index -> window workspace tensor
        self._epoch = 0

    def __del__(self):
        if getattr(self, "_handles", None) is not None:
            self._handles.destroy_all()

    def invalidate(self) -> None:
        """Force a weight reload on the next call (after in-place writes through `.data`, which torch does not version)."""
        self._epoch += 1

    def _fingerprint(self):
        return (self._epoch,) + tuple((p.data_ptr(), p._version) for p in self.parameters())

    def _handle(self, device: torch.device):
        return self._handles.get(device, self._fingerprint(), self._create, self._load)

    def _load_layers(self, entry: str, h, device: torch.device) -> None:
        """entry(h, weights, biases, stream) on the folded weights and the biases of self._layers (a GAN vocoder's
        weight-normalised convolutions in state_dict order)."""
        ws = [m.folded().to(device).contiguous() for m in self._layers]
        bs = [m.bias.detach().float().to(device).contiguous() for m in self._layers]
        wp = (C.c_void_p * len(ws))(*[t.data_ptr() for t in ws])
        bp = (C.c_void_p * len(bs))(*[t.data_ptr() for t in bs])
        _lib.check(getattr(_lib.load(), entry)(h, wp, bp, _lib.stream_ptr(device)), entry)

    def _workspace(self, h, B: int, L: int, device: torch.device) -> torch.Tensor:
        return workspace(self._ws, device, query_bytes(f"fs2_{self._NAME}_workspace_bytes", h, B, L))

    def _status_table(self):
        """[(bit, message)] of the status word: FS2_<_NAME>_BAD_LENGTH, _BAD_START where the vocoder has windows, _RANGE."""
        status = "FS2_" + self._NAME.upper()
        table = [(getattr(_lib, status + "_BAD_LENGTH"), "every olens[b] must lie in [1, Lmax]")]
        if hasattr(_lib, status + "_BAD_START"):
            table.append((getattr(_lib, status + "_BAD_START"), "every starts[b] must be >= 0"))
        table.append((getattr(_lib, status + "_RANGE"),
                      f"activations exceed the range of the fp16 operand planes in math_mode={self.math_mode!r} "
                      f"(some GEMM input above {65504 / 16:g} in magnitude); use math_mode='fp32' or 'tf32'"))
        return table

    def _check_status(self, status: torch.Tensor) -> None:
        check_status(status, self._status_table())

    @staticmethod
    def _check_mels_olens(mels, olens) -> None:
        """The checks of mels [B, Lmax, 80] and olens [B] that need no device."""
        if not torch.is_tensor(mels) or mels.dim() != 3 or mels.shape[2] != N_MELS or mels.shape[0] == 0 or mels.shape[1] == 0:
            raise ValueError(f"mels must be a non-empty [B, Lmax, {N_MELS}] tensor")
        if not torch.is_tensor(olens) or olens.dim() != 1 or olens.shape[0] != mels.shape[0]:
            raise ValueError(f"olens must be a [B={mels.shape[0]}] tensor")
        if olens.dtype.is_floating_point or olens.dtype == torch.bool:
            raise ValueError("olens must be an integer tensor")

    def _mels_olens(self, mels, olens, check_size=None):
        """Validated (mels fp32, olens int64, B, Lmax) of a call whose only inputs they are.  check_size(B, Lmax): the
        limits (default: the whole call's)."""
        self._check_mels_olens(mels, olens)
        if not mels.is_cuda or not olens.is_cuda:
            raise ValueError("mels and olens must be CUDA tensors (the H100 path has no CPU fallback)")
        B, L, _ = mels.shape
        (check_size or self._check_size)(B, L)
        return mels.to(torch.float32).contiguous(), olens.to(device=mels.device, dtype=torch.int64).contiguous(), B, L

    def _check_rows(self, rows: int, formula: str, noun: str, where: str, advice: str) -> None:
        """The limits the C entries put on the rows of their largest buffer, raised here as ValueError: below 2^31, and at
        most 65535 * 128 in fp32 mode (its CUDA-core GEMMs put 128-row tiles on grid.y)."""
        if rows >= 1 << 31:
            raise ValueError(f"{formula} must stay below 2^31 {noun} rows ({where})")
        if self.math_mode == "fp32" and rows > 65535 * 128:
            raise ValueError(f"math_mode='fp32' takes at most 65535 * 128 {noun} rows, {formula} = {rows} ({where}); {advice}")

    def _check_size(self, B: int, L: int) -> None:
        """_check_rows on the whole call's rows."""
        self._check_rows(*self._rows(B, L), f"B={B}, Lmax={L}", "split the batch or use another math mode")

    def _whole(self, call, mels, olens, B: int, L: int):
        """The whole call on validated mels / olens: -> (audio [B, Lmax * HOP], alens = olens * HOP)."""
        dev = mels.device
        h = self._handle(dev)
        ws = self._workspace(h, B, L, dev)
        audio = torch.empty((B, L * self.HOP), dtype=torch.float32, device=dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            call(h, mels, olens, B, L, audio, status, ws)
        self._check_status(status)
        return audio, olens * self.HOP

    def _call(self, h, mels, olens, B: int, L: int, audio: torch.Tensor, status: torch.Tensor, ws: torch.Tensor) -> None:
        """The whole call of an upsampling chain: fs2_<_NAME>."""
        name = f"fs2_{self._NAME}"
        _lib.check(getattr(_lib.load(), name)(h, _lib.ptr(mels), _lib.ptr(olens), B, L, _lib.ptr(audio), _lib.ptr(status), _lib.ptr(ws),
                                              ws.numel(), _lib.stream_ptr(mels.device)), name)

    def forward(self, mels: torch.Tensor, olens: torch.Tensor, chunk_frames: int | None = None):
        """-> (audio [B, Lmax * 256] fp32, alens [B] int64 = olens * 256).

        chunk_frames=k: the same bits, computed as windows of k frames written straight into the output, with the
        workspace of one window (fs2_<_NAME>_window): in fp32 mode this vocodes batches the whole call refuses.  Still one
        host read per call: the windows' status words are ORed on the device."""
        if chunk_frames is not None:
            mels, olens, B, L = self._window_inputs(mels, olens, chunk_frames)
            return self._chunked(self._window_call, mels, olens, B, L, chunk_frames)
        mels, olens, B, L = self._mels_olens(mels, olens)
        return self._whole(self._call, mels, olens, B, L)

    # ---- windows (MelGAN, HiFi-GAN and WaveGlow) ------------------------------------------------------------------
    def _window_workspace(self, h, B: int, n_frames: int, device: torch.device) -> torch.Tensor:
        return workspace(self._wws, device, query_bytes(f"fs2_{self._NAME}_window_workspace_bytes", h, B, n_frames))

    @staticmethod
    def _check_frames(n_frames) -> None:
        if isinstance(n_frames, bool) or not isinstance(n_frames, int) or n_frames < 1:
            raise ValueError(f"n_frames / chunk_frames must be an int >= 1 (got {n_frames!r})")

    def _check_window_size(self, B: int, n_frames: int) -> None:
        """_check_rows on a window's rows."""
        self._check_frames(n_frames)
        self._check_rows(*self._window_rows(B, n_frames), "window", f"B={B}, n_frames={n_frames}", "use fewer frames per window")

    def _check_extent(self, L: int, rate: int = HOP, noun: str = "samples") -> None:
        """A window's limit on Lmax, which bounds only the per-utterance rows: (Lmax + _TAIL) * rate below 2^31."""
        if (L + self._TAIL) * rate >= 1 << 31:
            lmax = f"(Lmax + {self._TAIL})" if self._TAIL else "Lmax"
            raise ValueError(f"{lmax} * {rate} must stay below 2^31 {noun} (Lmax={L})")

    def _window_rows(self, B: int, n_frames: int):
        """An upsampling chain's largest window buffer: B * (up_s * n_frames + 2 h_s) rows for the level s with the most."""
        rates, R, margin0, *post = self._chain()
        ups = itertools.accumulate(rates, operator.mul, initial=1)
        n, up, h = max((up * n_frames + 2 * h, up, h) for up, h in zip(ups, ups_window_plan(rates, R, margin0, *post)["halo"]))
        return B * n, f"B * ({up} * n_frames + {2 * h})"

    def _window_inputs(self, mels, olens, n_frames):
        """_mels_olens with the window's limits in place of the whole call's."""
        self._check_frames(n_frames)

        def check(B, L):
            self._check_window_size(B, n_frames)
            self._check_extent(L)
        return self._mels_olens(mels, olens, check)

    def _window_call(self, h, mels, olens, starts, B: int, L: int, n_frames: int, audio: torch.Tensor, ld: int, status: torch.Tensor,
                     ws: torch.Tensor) -> None:
        """A window call of an upsampling chain: fs2_<_NAME>_window."""
        name, dev = f"fs2_{self._NAME}_window", mels.device
        with torch.cuda.device(dev):
            _lib.check(getattr(_lib.load(), name)(h, _lib.ptr(mels), _lib.ptr(olens), _lib.ptr(starts), B, L, n_frames, audio.data_ptr(), ld,
                                                  _lib.ptr(status), _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev)), name)

    def window(self, mels: torch.Tensor, olens: torch.Tensor, starts, n_frames: int):
        """One window of the audio (DESIGN.md sections 11 and 17): -> (audio [B, n_frames * 256] fp32, alens [B] int64 =
        clamp(olens - starts, 0, n_frames) * 256).  audio[b, :alens[b]] are samples [starts[b] * 256, ...) of
        `forward(mels, olens)[0][b]`, bit for bit; the rest is 0.  starts: an int (every utterance), a host list or tensor,
        or a device tensor.  Only mel frames [starts[b] - r, starts[b] + n_frames + r) below olens[b] are read, r = the
        first upsampling's reach + 3 (6 for MelGAN, 13 for HiFi-GAN V1, 11 for V3); the workspace depends on B and
        n_frames only.  One host read per call."""
        mels, olens, B, L = self._window_inputs(mels, olens, n_frames)
        return self._window(self._window_call, mels, olens, starts, B, L, n_frames)

    def stream(self, mels: torch.Tensor, olens: torch.Tensor, chunk_frames: int = 32):
        """Lockstep windows: yields (audio, alens) of `window(mels, olens, k * chunk_frames, chunk_frames)` for k = 0 ..
        ceil(Lmax / chunk_frames) - 1, the last one cut at Lmax, so that the chunks concatenated along time are
        `forward(mels, olens)`.  Utterances that have ended give rows of 0 (alens 0)."""
        self._check_frames(chunk_frames)
        yield from self._stream(mels, chunk_frames, lambda c0, n: self.window(mels, olens, c0, n))

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

    def _window(self, call, mels, olens, starts, B: int, L: int, n_frames: int):
        """One window on validated mels / olens: -> (audio [B, n_frames * HOP], alens)."""
        dev = mels.device
        starts = self._starts(starts, B, dev)
        h = self._handle(dev)
        ws = self._window_workspace(h, B, n_frames, dev)
        audio = torch.empty((B, n_frames * self.HOP), dtype=torch.float32, device=dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        call(h, mels, olens, starts, B, L, n_frames, audio, n_frames * self.HOP, status, ws)
        self._check_status(status)
        return audio, (olens - starts).clamp(0, n_frames) * self.HOP

    @staticmethod
    def _stream(mels, chunk_frames: int, window):
        """window(c0, n) for the lockstep windows c0 = 0, chunk_frames, ... of mels' Lmax frames, the last one cut at Lmax."""
        L = mels.shape[1]
        for c0 in range(0, L, chunk_frames):
            yield window(c0, min(chunk_frames, L - c0))

    def _chunked(self, call, mels, olens, B: int, L: int, k: int):
        """forward(chunk_frames=k) on validated mels / olens: windows of k frames written straight into the output, one
        host read for all of them (their status words are ORed on the device)."""
        dev = mels.device
        h = self._handle(dev)
        ws = self._window_workspace(h, B, min(k, L), dev)
        audio = torch.empty((B, L * self.HOP), dtype=torch.float32, device=dev)
        c0s = list(range(0, L, k))
        starts = torch.tensor(c0s, dtype=torch.int64).repeat_interleave(B).reshape(len(c0s), B).to(dev)
        status = torch.empty((len(c0s),), dtype=torch.int32, device=dev)
        for i, c0 in enumerate(c0s):
            n = min(k, L - c0)
            call(h, mels, olens, starts[i], B, L, n, audio[:, c0 * self.HOP:], L * self.HOP, status[i: i + 1], ws)
        bits = torch.tensor([bit for bit, _ in self._status_table()], dtype=torch.int32, device=dev)
        self._check_status(((status[:, None] & bits) != 0).any(0).int().mul(bits).sum().reshape(1))
        return audio, olens * self.HOP
