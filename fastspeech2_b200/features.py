"""Training features on the device (DESIGN.md section 14): what the reference's nvidia_preprocessing.py computes per wav
file (utils/stft.py:188-204, nvidia_preprocessing.py:39, dataset/audio_processing.py:54-70), for a ragged batch.

For wavs [B, Nmax] fp32 on the GPU with lens [B] (integer), utterance b is wavs[b, :lens[b]]; samples past lens[b] are
never read.  With T_b = lens[b] // hop + 1 and Tmax = Nmax // hop + 1:

  mels   [B, Tmax, n_mels] fp32   log(max(mel_basis . |STFT(x_b)|, 1e-5)), the layout `synthesize` returns
  energy [B, Tmax] fp32           sqrt(sum_c |STFT(x_b)|[c]^2)  (torch.norm(mag, dim=0))
  flens  [B] int64                T_b
  f0     [B, Tmax] float64        pyworld.dio(float64(x_b), sample_rate, f0_floor, f0_ceil, channels_in_octave,
                                  frame_period = hop / sample_rate * 1000, speed = 1, allowed_range)[:plens[b]]
  plens  [B] int64                min(f0_length_b, T_b)

Everything past T_b / plens[b] is +0, and utterance b is bit-identical to a B = 1 call on its own samples.  The STFT and
mel filterbank run on the library's tap GEMM in `math_mode` ("3xf16" by default, fp32-class; also "fp32", "tf32",
"f16"); DIO runs in float64 on the CUDA cores.  One host read per call (the device-side length and range checks)."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._kernel_module import Handles, check_status, query_bytes, workspace
from .vocoder import STFT, mel_filterbank


class FeatureExtractor(torch.nn.Module):
    def __init__(self, sample_rate: int = 22050, n_fft: int = 1024, hop_length: int = 256, win_length: int = 1024,
                 n_mels: int = 80, fmin: float = 0.0, fmax=8000.0, math_mode: str = "3xf16", f0_floor: float = 71.0,
                 f0_ceil: float = 800.0, channels_in_octave: float = 2.0, allowed_range: float = 0.1):
        super().__init__()
        if math_mode not in _lib.MATH_MODES:
            raise ValueError(f"math_mode must be one of {sorted(_lib.MATH_MODES)}")
        self.sample_rate, self.n_fft, self.hop_length, self.win_length = int(sample_rate), int(n_fft), int(hop_length), int(win_length)
        self.n_mels, self.fmin, self.fmax, self.math_mode = int(n_mels), float(fmin), fmax, math_mode
        self.f0_floor, self.f0_ceil = float(f0_floor), float(f0_ceil)
        self.channels_in_octave, self.allowed_range = float(channels_in_octave), float(allowed_range)
        self.frame_period = self.hop_length / self.sample_rate * 1000     # the reference's expression, in this order
        self.cutoff = self.n_fft // 2 + 1
        self.stft = STFT(self.n_fft, self.hop_length, self.win_length, math_mode=math_mode)   # the windowed Fourier basis
        self.register_buffer("mel_basis", torch.from_numpy(mel_filterbank(self.sample_rate, self.n_fft, self.n_mels, self.fmin, fmax)))
        self._sizer = None          # an fs2_features* that is never loaded: answers workspace queries without a device
        self._handles = Handles("fs2_features_destroy")   # keyed by the data pointers the weights were loaded from
        self._ws = {}               # device index -> workspace tensor

    @classmethod
    def from_hp(cls, hp, math_mode: str = "3xf16") -> "FeatureExtractor":
        """Audio parameters from `hp.audio` (configs/default.yaml): sample_rate, n_fft, hop_length, win_length, n_mels (or
        num_mels), fmin, fmax.  DIO uses the reference's pyworld defaults."""
        a = hp["audio"] if isinstance(hp, dict) else hp.audio
        n_mels = a["n_mels"] if "n_mels" in a else a["num_mels"]
        return cls(a["sample_rate"], a["n_fft"], a["hop_length"], a["win_length"], n_mels, a["fmin"], a["fmax"], math_mode=math_mode)

    def __del__(self):
        if getattr(self, "_handles", None) is not None:
            self._handles.destroy_all()
        lib = _lib._lib
        if lib is not None and getattr(self, "_sizer", None):
            lib.fs2_features_destroy(self._sizer)

    def _config(self) -> _lib.FeaturesConfig:
        return _lib.FeaturesConfig(self.sample_rate, self.n_fft, self.hop_length, self.win_length, self.n_mels,
                                   _lib.MATH_MODES[self.math_mode], self.f0_floor, self.f0_ceil, self.channels_in_octave,
                                   self.allowed_range)

    def _create(self):
        h = C.c_void_p()
        _lib.check(_lib.load().fs2_features_create(C.byref(h), C.byref(self._config())), "fs2_features_create")
        return h.value

    def workspace_bytes(self, B: int, n_max: int) -> int:
        """Bytes of device workspace a call on [B, n_max] samples needs (either entry)."""
        if self._sizer is None:
            self._sizer = self._create()
        return query_bytes("fs2_features_workspace_bytes", self._sizer, int(B), int(n_max))

    def _handle(self, device: torch.device):
        return self._handles.get(device, tuple(t.data_ptr() for t in (self.stft.forward_basis, self.mel_basis)), self._create, self._load)

    def _load(self, h, device: torch.device) -> None:
        w = [t.to(device=device, dtype=torch.float32).contiguous() for t in (self.stft.forward_basis, self.mel_basis)]
        _lib.check(_lib.load().fs2_features_load(h, _lib.ptr(w[0]), _lib.ptr(w[1]), _lib.stream_ptr(device)), "fs2_features_load")

    def _workspace(self, B: int, n_max: int, device: torch.device) -> torch.Tensor:
        return workspace(self._ws, device, self.workspace_bytes(B, n_max))

    def _inputs(self, wavs: torch.Tensor, lens: torch.Tensor):
        if not torch.is_tensor(wavs) or wavs.dim() != 2 or wavs.shape[0] == 0:
            raise ValueError("wavs must be a non-empty [B, Nmax] tensor")
        if wavs.dtype != torch.float32:
            raise ValueError(f"wavs must be float32 (got {wavs.dtype})")
        if not torch.is_tensor(lens) or lens.dim() != 1 or lens.shape[0] != wavs.shape[0]:
            raise ValueError(f"lens must be a [B={wavs.shape[0]}] tensor")
        if lens.dtype.is_floating_point or lens.dtype.is_complex or lens.dtype == torch.bool:
            raise ValueError("lens must be an integer tensor")
        B, n_max = wavs.shape
        if n_max <= self.n_fft // 2:
            raise ValueError(f"Nmax={n_max} samples is too short: reflect padding needs more than n_fft/2 = {self.n_fft // 2}")
        if not wavs.is_cuda or not lens.is_cuda:
            raise ValueError("wavs and lens must be CUDA tensors (the H100 path has no CPU fallback)")
        return wavs.contiguous(), lens.to(device=wavs.device, dtype=torch.int64).contiguous(), B, n_max

    def _check_status(self, status: torch.Tensor) -> None:
        check_status(status, [
            (_lib.FS2_FEAT_BAD_LENGTH, f"every lens[b] must lie in (n_fft/2, Nmax] = ({self.n_fft // 2}, Nmax] (reflect padding at "
                                       f"the utterance's edges)"),
            (_lib.FS2_FEAT_RANGE, "samples must lie in [-1, 1] (the reference asserts it before its STFT)")])

    def _call(self, entry: str, wavs, lens, outs):
        dev = wavs.device
        h = self._handle(dev)
        ws = self._workspace(wavs.shape[0], wavs.shape[1], dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(getattr(_lib.load(), entry)(h, _lib.ptr(wavs), _lib.ptr(lens), wavs.shape[0], wavs.shape[1],
                                                   *[_lib.ptr(t) for t in outs], _lib.ptr(status), _lib.ptr(ws), ws.numel(),
                                                   _lib.stream_ptr(dev)), entry)
        return status

    def mel_energy(self, wavs: torch.Tensor, lens: torch.Tensor):
        """-> (mels [B, Tmax, n_mels] fp32, energy [B, Tmax] fp32, flens [B] int64)."""
        wavs, lens, B, n_max = self._inputs(wavs, lens)
        T = n_max // self.hop_length + 1
        mels = torch.empty((B, T, self.n_mels), dtype=torch.float32, device=wavs.device)
        energy = torch.empty((B, T), dtype=torch.float32, device=wavs.device)
        self._check_status(self._call("fs2_mel_energy", wavs, lens, (mels, energy)))
        return mels, energy, lens // self.hop_length + 1

    def pitch(self, wavs: torch.Tensor, lens: torch.Tensor):
        """-> (f0 [B, Tmax] float64, plens [B] int64)."""
        wavs, lens, B, n_max = self._inputs(wavs, lens)
        T = n_max // self.hop_length + 1
        f0 = torch.empty((B, T), dtype=torch.float64, device=wavs.device)
        plens = torch.empty((B,), dtype=torch.int64, device=wavs.device)
        self._check_status(self._call("fs2_dio", wavs, lens, (f0, plens)))
        return f0, plens

    def forward(self, wavs: torch.Tensor, lens: torch.Tensor):
        """-> (mels, energy, flens, f0, plens)."""
        mels, energy, flens = self.mel_energy(wavs, lens)
        f0, plens = self.pitch(wavs, lens)
        return mels, energy, flens, f0, plens
