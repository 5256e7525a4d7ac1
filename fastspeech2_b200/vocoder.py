"""Vocoder hand-off on the device (SURVEY.md section 8f-2): the STFT / inverse-STFT pair and the Griffin-Lim loop the
reference falls back to when no neural vocoder is configured (inference.py:188-193 -> utils/stft.py:41-156,
dataset/audio_processing.py:224-240).

Same class surface as the reference's `STFT` (`transform`, `inverse`, `forward`, buffers `forward_basis` / `inverse_basis`
built the same way: windowed real/imag Fourier rows and their scaled pseudo-inverse), but the arithmetic runs on
libfs2b200.so: the reference's strided `F.conv1d` / `F.conv_transpose1d` are GEMMs over a [frames, n_fft] matrix, issued
through the library's tap-GEMM (fp32-class 3xF16 on tensor-core by default) with hand-written kernels for reflect-padding +
framing, magnitude / phase, recombination and overlap-add + window-sum normalisation (csrc/stft.cu).  No cuFFT, no torch
compute.  Everything stays on the GPU between the mel batch and the waveform (the reference round-trips through `.cpu()`
every iteration, utils/stft.py:97-103).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from ._kernel_module import Handles, check_status, query_bytes, workspace


def _hann(win_length: int, n_fft: int) -> np.ndarray:
    """scipy.signal.get_window("hann", win_length, fftbins=True) zero-padded to n_fft about its centre (librosa pad_center)."""
    w = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(win_length) / win_length)
    lpad = (n_fft - win_length) // 2
    return np.pad(w, (lpad, n_fft - win_length - lpad))


def window_sumsquare(n_frames: int, hop_length: int, win_length: int, n_fft: int) -> np.ndarray:
    """dataset/audio_processing.py:169-221 (librosa 0.6): sum of squared windows at every sample, float32."""
    n = n_fft + hop_length * (n_frames - 1)
    x = np.zeros(n, dtype=np.float32)
    win_sq = _hann(win_length, n_fft) ** 2
    for i in range(n_frames):
        s = i * hop_length
        x[s: min(n, s + n_fft)] += win_sq[: max(0, min(n_fft, n - s))]
    return x


class STFT(torch.nn.Module):
    """Drop-in for utils/stft.py:41-156 (hann window only), on the H100 kernels.  `math_mode`: "3xf16" (default,
    fp32-class), "fp32" (CUDA cores) or "f16" / "tf32" for the two GEMMs."""

    def __init__(self, filter_length: int = 800, hop_length: int = 200, win_length: int = 800, window: str = "hann", math_mode: str = "3xf16"):
        super().__init__()
        if window != "hann":
            raise NotImplementedError("only the hann window the reference uses is implemented")
        assert filter_length >= win_length and filter_length % 80 == 0 or filter_length % 128 == 0, "n_fft must be a multiple of 80 or 128 (GEMM tile widths)"
        self.filter_length, self.hop_length, self.win_length, self.window = filter_length, hop_length, win_length, window
        self.math_mode = _lib.MATH_MODES[math_mode]
        scale = filter_length / hop_length
        fourier = np.fft.fft(np.eye(filter_length))
        self.cutoff = cutoff = filter_length // 2 + 1
        fourier = np.vstack([np.real(fourier[:cutoff, :]), np.imag(fourier[:cutoff, :])])          # [2*cutoff, n_fft]
        win = _hann(win_length, filter_length)
        fwd = torch.FloatTensor(fourier[:, None, :]) * torch.from_numpy(win).float()
        inv = torch.FloatTensor(np.linalg.pinv(scale * fourier).T[:, None, :]) * torch.from_numpy(win).float()
        self.register_buffer("forward_basis", fwd.float())                                         # [2*cutoff, 1, n_fft]
        self.register_buffer("inverse_basis", inv.float())
        # GEMM operands in the library's [taps=1][N][K] layout, N / K padded with zero rows / columns to the next tile multiple
        self.cpad = (2 * cutoff + 63) // 64 * 64
        w_f = torch.zeros(self.cpad, filter_length); w_f[: 2 * cutoff] = fwd[:, 0, :]
        w_i = torch.zeros(filter_length, self.cpad); w_i[:, : 2 * cutoff] = inv[:, 0, :].T
        self.register_buffer("_w_forward", w_f.contiguous(), persistent=False)
        self.register_buffer("_w_inverse", w_i.contiguous(), persistent=False)
        self.register_buffer("_zero_bias_f", torch.zeros(self.cpad), persistent=False)
        self.register_buffer("_zero_bias_i", torch.zeros(filter_length), persistent=False)
        self._wsum = {}

    def _gemm(self, x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
        B, L, K = x.shape
        N = w.shape[0]
        out = torch.empty((B, L, N), dtype=torch.float32, device=x.device)
        _lib.check(_lib.load().fs2_op_tap_gemm(self.math_mode, _lib.ptr(x), B, L, K, _lib.ptr(w), _lib.ptr(bias), N, 1, 0, None, _lib.ptr(out),
                                               _lib.stream_ptr(x.device)), "fs2_op_tap_gemm")
        return out

    def transform(self, input_data: torch.Tensor):
        """[B, n] samples -> (magnitude, phase), each [B, n_fft/2+1, frames] (utils/stft.py:82-112)."""
        lib = _lib.load()
        x = input_data.to(dtype=torch.float32).contiguous()
        if not x.is_cuda:
            raise _lib.Fs2Error("STFT.transform: CUDA tensor required (no CPU fallback)")
        B, n = x.shape
        self.num_samples = n
        frames = n // self.hop_length + 1
        st = _lib.stream_ptr(x.device)
        fr = torch.empty((B, frames, self.filter_length), dtype=torch.float32, device=x.device)
        _lib.check(lib.fs2_stft_frames(_lib.ptr(x), B, n, self.filter_length, self.hop_length, frames, _lib.ptr(fr), st), "fs2_stft_frames")
        spec = self._gemm(fr, self._w_forward, self._zero_bias_f)
        mag = torch.empty((B, self.cutoff, frames), dtype=torch.float32, device=x.device)
        phase = torch.empty_like(mag)
        _lib.check(lib.fs2_stft_magphase(_lib.ptr(spec), self.cpad, B, self.cutoff, frames, _lib.ptr(mag), _lib.ptr(phase), st), "fs2_stft_magphase")
        return mag, phase

    def inverse(self, magnitude: torch.Tensor, phase: torch.Tensor) -> torch.Tensor:
        """(magnitude, phase) [B, cutoff, frames] -> [B, 1, (frames-1)*hop] samples (utils/stft.py:114-151)."""
        lib = _lib.load()
        mag, ph = magnitude.to(torch.float32).contiguous(), phase.to(torch.float32).contiguous()
        if not mag.is_cuda:
            raise _lib.Fs2Error("STFT.inverse: CUDA tensors required (no CPU fallback)")
        B, cutoff, frames = mag.shape
        assert cutoff == self.cutoff, f"expected {self.cutoff} frequency rows, got {cutoff}"
        st = _lib.stream_ptr(mag.device)
        rec = torch.empty((B, frames, self.cpad), dtype=torch.float32, device=mag.device)
        _lib.check(lib.fs2_istft_recombine(_lib.ptr(mag), _lib.ptr(ph), B, cutoff, frames, self.cpad, _lib.ptr(rec), st), "fs2_istft_recombine")
        fr = self._gemm(rec, self._w_inverse, self._zero_bias_i)
        key = (frames, str(mag.device))
        if key not in self._wsum:
            self._wsum[key] = torch.from_numpy(window_sumsquare(frames, self.hop_length, self.win_length, self.filter_length)).to(mag.device)
        y = torch.empty((B, 1, (frames - 1) * self.hop_length), dtype=torch.float32, device=mag.device)
        _lib.check(lib.fs2_istft_overlap_add(_lib.ptr(fr), B, self.filter_length, self.hop_length, frames, _lib.ptr(self._wsum[key]),
                                             float(np.finfo(np.float32).tiny), _lib.ptr(y), st), "fs2_istft_overlap_add")
        return y

    def forward(self, input_data: torch.Tensor) -> torch.Tensor:
        self.magnitude, self.phase = self.transform(input_data)
        return self.inverse(self.magnitude, self.phase)


def griffin_lim(magnitudes: torch.Tensor, stft_fn: STFT, n_iters: int = 30, angles: torch.Tensor = None) -> torch.Tensor:
    """dataset/audio_processing.py:224-240: random initial phases, then n_iters x (transform -> keep phase -> inverse).
    `angles` may be given for reproducibility (the reference draws them with np.random)."""
    if angles is None:
        angles = np.angle(np.exp(2j * np.pi * np.random.rand(*magnitudes.size()))).astype(np.float32)
        angles = torch.from_numpy(angles)
    angles = angles.to(magnitudes.device)
    signal = stft_fn.inverse(magnitudes, angles).squeeze(1)
    for _ in range(n_iters):
        _, angles = stft_fn.transform(signal)
        signal = stft_fn.inverse(magnitudes, angles).squeeze(1)
    return signal


# ---- batched waveform synthesis: mel inversion + per-utterance Griffin-Lim (DESIGN.md section 7) ----------------------

def _hz_to_mel(f):
    """Slaney mel scale (librosa 0.7 `hz_to_mel`, htk=False): linear below 1 kHz, logarithmic above."""
    f = np.asanyarray(f, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, min_log_hz) / min_log_hz) / logstep, f / f_sp)


def _mel_to_hz(m):
    m = np.asanyarray(m, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_filterbank(sample_rate: int, n_fft: int, n_mels: int = 128, fmin: float = 0.0, fmax=None) -> np.ndarray:
    """librosa 0.7 `filters.mel(sr, n_fft, n_mels, fmin, fmax)` (htk=False, Slaney area normalisation), the matrix the
    reference's `TacotronSTFT` builds: float32 [n_mels, n_fft/2+1].  Triangles on the Slaney mel scale between n_mels + 2
    equally spaced mel points, each scaled by 2 / (its bandwidth in Hz)."""
    fmax = float(sample_rate) / 2 if fmax is None else float(fmax)
    weights = np.zeros((n_mels, 1 + n_fft // 2), dtype=np.float32)
    fftfreqs = np.linspace(0, float(sample_rate) / 2, 1 + n_fft // 2, endpoint=True)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    weights *= (2.0 / (mel_f[2: n_mels + 2] - mel_f[:n_mels]))[:, None]
    return weights


def mel_inverse(mel_basis: np.ndarray) -> np.ndarray:
    """P = pinv(mel_basis) in float64, rounded to float32: [n_fft/2+1, n_mels]."""
    return np.linalg.pinv(mel_basis.astype(np.float64)).astype(np.float32)


class GriffinLimVocoder(torch.nn.Module):
    """Batched log-mel -> waveform on the library's kernels (not in the reference, whose Griffin-Lim fallback receives
    log-mels where it needs linear magnitudes).  For mels [B, Lmax, n_mels] (what `FeedForwardTransformer.synthesize`
    returns) and frame counts olens [B]:

      M[b, f] = max(0, P . exp(mels[b, f]))  for f < olens[b]          (`mel_to_magnitude`, P = pinv(mel filterbank))
      audio[b] = Griffin-Lim of M[b] over its own olens[b] frames     (`__call__`)

    Each utterance's audio, audio[b, :alens[b]] with alens[b] = (olens[b] - 1) * hop, is bit-identical to a B = 1 call on
    its own frames with the same seed (or its slice of `angles`), whatever else is in the batch; audio past alens[b] is 0.
    Mel frames past olens[b] are never read.  `momentum` is the "fast Griffin-Lim" extrapolation (0: the reference's
    algorithm; 0.99: torchaudio's fast variant).  math_mode: "3xf16" (default, fp32-class), "fp32", "f16" or "tf32" for the
    three GEMMs, as in `STFT`.  One host read per call (the device-side length and range checks)."""

    def __init__(self, sample_rate: int = 22050, n_fft: int = 1024, hop_length: int = 256, win_length: int = 1024,
                 n_mels: int = 80, fmin: float = 0.0, fmax=8000.0, math_mode: str = "3xf16"):
        super().__init__()
        if math_mode not in _lib.MATH_MODES:
            raise ValueError(f"math_mode must be one of {sorted(_lib.MATH_MODES)}")
        self.sample_rate, self.n_fft, self.hop_length, self.win_length = int(sample_rate), int(n_fft), int(hop_length), int(win_length)
        self.n_mels, self.fmin, self.fmax, self.math_mode = int(n_mels), float(fmin), fmax, math_mode
        self.stft = STFT(self.n_fft, self.hop_length, self.win_length, math_mode=math_mode)   # the Fourier bases
        self.cutoff = self.stft.cutoff
        basis = mel_filterbank(self.sample_rate, self.n_fft, self.n_mels, self.fmin, fmax)
        self.register_buffer("mel_basis", torch.from_numpy(basis))                                  # [n_mels, cutoff]
        self.register_buffer("mel_inverse", torch.from_numpy(mel_inverse(basis)))                   # [cutoff, n_mels]
        self.register_buffer("_window_sq", torch.from_numpy(_hann(self.win_length, self.n_fft) ** 2).float(), persistent=False)
        self._handles = Handles("fs2_vocoder_destroy")   # keyed by the data pointers the bases were loaded from
        self._ws = {}            # device index -> workspace tensor

    @classmethod
    def from_hp(cls, hp, math_mode: str = "3xf16") -> "GriffinLimVocoder":
        """Audio parameters from `hp.audio` (configs/default.yaml): sample_rate, n_fft, hop_length, win_length, n_mels
        (or num_mels), fmin, fmax."""
        a = hp["audio"] if isinstance(hp, dict) else hp.audio
        n_mels = a["n_mels"] if "n_mels" in a else a["num_mels"]
        return cls(a["sample_rate"], a["n_fft"], a["hop_length"], a["win_length"], n_mels, a["fmin"], a["fmax"], math_mode=math_mode)

    def __del__(self):
        if getattr(self, "_handles", None) is not None:
            self._handles.destroy_all()

    def _bases(self):
        return (self.stft.forward_basis, self.stft.inverse_basis, self.mel_inverse, self._window_sq)

    def _handle(self, device: torch.device):
        return self._handles.get(device, tuple(t.data_ptr() for t in self._bases()), self._create, self._load)

    def _create(self):
        h = C.c_void_p()
        cfg = _lib.VocoderConfig(self.n_fft, self.hop_length, self.win_length, self.n_mels, _lib.MATH_MODES[self.math_mode])
        _lib.check(_lib.load().fs2_vocoder_create(C.byref(h), C.byref(cfg)), "fs2_vocoder_create")
        return h.value

    def _load(self, h, device: torch.device) -> None:
        bases = [t.to(device=device, dtype=torch.float32).contiguous() for t in self._bases()]
        _lib.check(_lib.load().fs2_vocoder_load(h, *[_lib.ptr(t) for t in bases], _lib.stream_ptr(device)), "fs2_vocoder_load")

    def _workspace(self, h, B: int, L: int, device: torch.device) -> torch.Tensor:
        return workspace(self._ws, device, query_bytes("fs2_vocoder_workspace_bytes", h, B, L))

    def _inputs(self, mels: torch.Tensor, olens: torch.Tensor, check_device: bool = True):
        if not torch.is_tensor(mels) or mels.dim() != 3 or mels.shape[2] != self.n_mels:
            raise ValueError(f"mels must be a [B, Lmax, n_mels={self.n_mels}] tensor")
        if not torch.is_tensor(olens) or olens.dim() != 1 or olens.shape[0] != mels.shape[0] or olens.shape[0] == 0:
            raise ValueError(f"olens must be a non-empty [B={mels.shape[0]}] tensor")
        if olens.dtype.is_floating_point or olens.dtype == torch.bool:
            raise ValueError("olens must be an integer tensor")
        B, L, _ = mels.shape
        if (L - 1) * self.hop_length <= self.n_fft // 2:
            raise ValueError(f"Lmax={L} frames is too short: reflect padding needs (olens[b]-1)*hop > n_fft/2")
        if check_device:
            self._on_device(mels, olens)
        return mels.to(torch.float32).contiguous(), olens.to(device=mels.device, dtype=torch.int64).contiguous(), B, L

    @staticmethod
    def _on_device(mels, olens):
        if not mels.is_cuda or not olens.is_cuda:
            raise ValueError("mels and olens must be CUDA tensors (the H100 path has no CPU fallback)")

    def _check_status(self, status: torch.Tensor) -> None:
        check_status(status, [
            (_lib.FS2_VOC_BAD_LENGTH, f"every olens[b] must lie in [1, Lmax] with (olens[b]-1)*hop > n_fft/2 = {self.n_fft // 2} "
                                      f"(reflect padding at the utterance's edges)"),
            (_lib.FS2_VOC_RANGE, f"magnitudes exceed the range of the fp16 operand planes in math_mode={self.math_mode!r} "
                                 f"(|exp(mel)|, |M| or |signal| above {65504 / 16:g}); use math_mode='fp32' or 'tf32'")])

    def mel_to_magnitude(self, mels: torch.Tensor, olens: torch.Tensor) -> torch.Tensor:
        """[B, Lmax, n_mels] log-mels -> linear magnitudes [B, n_fft/2+1, Lmax] (0 past olens[b]): the input `griffin_lim`
        and `STFT.inverse` take."""
        mels, olens, B, L = self._inputs(mels, olens)
        dev = mels.device
        h = self._handle(dev)
        ws = self._workspace(h, B, L, dev)
        mag = torch.empty((B, self.cutoff, L), dtype=torch.float32, device=dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.load().fs2_mel_magnitude(h, _lib.ptr(mels), _lib.ptr(olens), B, L, _lib.ptr(mag), _lib.ptr(status),
                                                     _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev)), "fs2_mel_magnitude")
        self._check_status(status)
        return mag

    def forward(self, mels: torch.Tensor, olens: torch.Tensor, *, n_iters: int = 30, momentum: float = 0.0, seed=0,
                angles: torch.Tensor = None):
        """-> (audio [B, (Lmax-1)*hop] fp32, alens [B] int64).  Initial phases: `angles` [B, n_fft/2+1, Lmax] (radians, the
        reference's layout), else uniform phases from Philox keyed by `seed` (an int, or a [B] tensor of per-utterance
        seeds) at counter f * (n_fft/2+1) + c."""
        if isinstance(n_iters, bool) or not isinstance(n_iters, int) or n_iters < 0:
            raise ValueError(f"n_iters must be an int >= 0 (got {n_iters!r})")
        momentum = float(momentum)
        if not (0.0 <= momentum < 1.0):
            raise ValueError(f"momentum must lie in [0, 1) (got {momentum})")
        mels_in, olens_in = mels, olens
        mels, olens, B, L = self._inputs(mels, olens, check_device=False)
        dev = mels.device
        seeds = None
        if angles is not None:
            if not torch.is_tensor(angles) or tuple(angles.shape) != (B, self.cutoff, L):
                raise ValueError(f"angles must be a [B={B}, {self.cutoff}, Lmax={L}] tensor")
            if not angles.is_cuda:
                raise ValueError("angles must be a CUDA tensor")
            angles = angles.to(device=dev, dtype=torch.float32).contiguous()
        elif torch.is_tensor(seed):
            if seed.dim() != 1 or seed.shape[0] != B or seed.dtype.is_floating_point or seed.dtype == torch.bool:
                raise ValueError(f"seed must be an int or a [B={B}] integer tensor")
            seeds = seed.to(device=dev, dtype=torch.int64).contiguous()
        elif isinstance(seed, int) and not isinstance(seed, bool):
            seeds = torch.full((B,), int(np.int64(np.uint64(seed % (1 << 64)))), dtype=torch.int64, device=dev)
        else:
            raise ValueError(f"seed must be an int or a [B={B}] integer tensor")
        self._on_device(mels_in, olens_in)
        h = self._handle(dev)
        ws = self._workspace(h, B, L, dev)
        audio = torch.empty((B, (L - 1) * self.hop_length), dtype=torch.float32, device=dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.load().fs2_griffin_lim(h, _lib.ptr(mels), _lib.ptr(olens), B, L, n_iters, momentum, _lib.ptr(seeds),
                                                   _lib.ptr(angles), _lib.ptr(audio), _lib.ptr(status), _lib.ptr(ws), ws.numel(),
                                                   _lib.stream_ptr(dev)), "fs2_griffin_lim")
        self._check_status(status)
        return audio, (olens - 1) * self.hop_length
