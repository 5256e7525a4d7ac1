"""Band-limited resampling on the GPU (DESIGN.md section 22): what the reference's preprocessing gets from
`librosa.load(path, sr=...)` for a file at another rate, for a ragged batch of mono utterances.

The reference pins librosa 0.7.0, which resamples with resampy 0.2.x (`res_type='kaiser_best'`) and then fixes the
length to ceil(N * ratio) samples.  `Resampler` restates that computation, and its output is bit-identical to the
float64 numpy restatement in oracle/resample_oracle.py.  Equality with librosa / resampy themselves holds by construction,
not by test.  resampy ships its filter table as a data file; `filter_table` rebuilds it with resampy's recipe, and
whether current numpy / scipy reproduce that file bit for bit is unverified.

Serving at another rate takes any vocoder's output as it is: `Resampler(22050, 48000)(*vocoder(mels, olens))`."""
from __future__ import annotations

import numpy as np
import scipy.signal
import torch
import torch.nn as nn

from . import _lib
from ._kernel_module import check_status, query_bytes, workspace

NUM_ZEROS = 64
NUM_TABLE = 512                                # table entries per zero crossing (resampy's precision 9)
ROLLOFF = 0.9475937167399596                   # resampy's kaiser_best
BETA = 14.769656459379492


def filter_table(orig_sr: int, new_sr: int) -> np.ndarray:
    """[32769, 2] float64: (win, delta) interleaved.  win is resampy's kaiser_best right wing, scaled by the ratio when
    downsampling; delta its forward difference after the scaling, 0 at the end."""
    n = NUM_TABLE * NUM_ZEROS
    sinc = ROLLOFF * np.sinc(ROLLOFF * np.linspace(0, NUM_ZEROS, num=n + 1, endpoint=True))
    win = scipy.signal.windows.kaiser(2 * n + 1, BETA)[n:] * sinc
    ratio = float(new_sr) / orig_sr
    if ratio < 1:
        win = win * ratio
    delta = np.zeros_like(win)
    delta[:-1] = np.diff(win)
    return np.ascontiguousarray(np.stack([win, delta], axis=1))


def out_length(n: int, orig_sr: int, new_sr: int) -> int:
    """ceil(n * ratio): the samples librosa returns for n input samples."""
    return int(np.ceil(n * (float(new_sr) / orig_sr)))


def workspace_bytes(B: int, Nmax: int, orig_sr: int, new_sr: int) -> int:
    """Bytes of device workspace a call on [B, Nmax] needs: the time register, 8 B per output sample."""
    return query_bytes("fs2_resample_workspace_bytes", int(B), int(Nmax), int(orig_sr), int(new_sr),
                       out_length(int(Nmax), orig_sr, new_sr))


def _rate(name: str, v) -> int:
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not 1 <= v <= 1 << 24:
        raise ValueError(f"{name} must be an integer sample rate in [1, 2^24] Hz (got {v!r})")
    return int(v)


class Resampler(nn.Module):
    """Resampler(orig_sr, new_sr): forward(wavs [B, Nmax] fp32, lens [B] int) -> (out [B, Mmax] fp32, olens [B] int64)
    with Mmax = ceil(Nmax * ratio) and olens[b] = ceil(lens[b] * ratio), out[b, olens[b]:] = +0, on CUDA tensors only.
    Samples at or past lens[b] are never read, and each utterance's output does not depend on its batch mates.  With
    orig_sr == new_sr it returns (wavs, lens as int64) unchanged, as librosa does, and runs nothing.  One host read per
    call; the filter table is built once and cached per device."""

    def __init__(self, orig_sr: int, new_sr: int):
        super().__init__()
        self.orig_sr, self.new_sr = _rate("orig_sr", orig_sr), _rate("new_sr", new_sr)
        if self.orig_sr != self.new_sr and int(min(1.0, float(self.new_sr) / self.orig_sr) * NUM_TABLE) < 1:
            raise ValueError(f"cannot downsample by more than {NUM_TABLE} ({self.orig_sr} -> {self.new_sr} Hz)")
        self._table = {}         # device index -> the table on that device
        self._ws = {}            # device index -> workspace tensor

    def extra_repr(self) -> str:
        return f"orig_sr={self.orig_sr}, new_sr={self.new_sr}"

    def forward(self, wavs: torch.Tensor, lens: torch.Tensor):
        if not torch.is_tensor(wavs) or wavs.dim() != 2 or min(wavs.shape) == 0:
            raise ValueError("wavs must be a non-empty [B, Nmax] tensor")
        if wavs.dtype != torch.float32:
            raise ValueError(f"wavs must be float32 (got {wavs.dtype})")
        B, N = wavs.shape
        if not torch.is_tensor(lens) or lens.dim() != 1 or lens.shape[0] != B:
            raise ValueError(f"lens must be a [B={B}] tensor")
        if lens.dtype.is_floating_point or lens.dtype.is_complex or lens.dtype == torch.bool:
            raise ValueError(f"lens must be an integer tensor (got {lens.dtype})")
        dev = wavs.device
        if not (wavs.is_cuda and lens.is_cuda and lens.device == dev):
            raise ValueError("wavs and lens must be CUDA tensors on one device (the H100 path has no CPU fallback)")
        lens = lens.to(torch.int64).contiguous()
        if self.orig_sr == self.new_sr:
            return wavs, lens
        M = out_length(N, self.orig_sr, self.new_sr)
        if M >= 1 << 26:
            raise ValueError(f"Nmax={N} gives {M} output samples; a call takes fewer than 2^26 (split the utterances)")
        wavs = wavs.contiguous()
        if dev.index not in self._table:
            self._table[dev.index] = torch.from_numpy(filter_table(self.orig_sr, self.new_sr)).to(dev)
        ws = workspace(self._ws, dev, workspace_bytes(B, N, self.orig_sr, self.new_sr))
        out = torch.empty((B, M), dtype=torch.float32, device=dev)
        olens = torch.empty(B, dtype=torch.int64, device=dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.load().fs2_resample(_lib.ptr(wavs), _lib.ptr(lens), B, N, _lib.ptr(self._table[dev.index]), self.orig_sr,
                                                self.new_sr, _lib.ptr(out), _lib.ptr(olens), M, _lib.ptr(status), _lib.ptr(ws),
                                                ws.numel(), _lib.stream_ptr(dev)), "fs2_resample")
        check_status(status, [
            (_lib.FS2_RS_BAD_LENGTH, f"every lens[b] must lie in [1, Nmax={N}] and give at least one output sample "
                                     f"(int(lens[b] * {self.new_sr} / {self.orig_sr}) >= 1)"),
            (_lib.FS2_RS_NONFINITE, "wavs must be finite within lens (found NaN or inf)")])
        return out, olens
