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

import torch
import torch.nn as nn

from . import _lib
from ._kernel_module import HOP, MAX_WAV_VALUE, N_MELS, NeuralVocoder, _WNConv, normalise_checkpoint, read_checkpoint

_STAGES = ((512, 256, 8), (256, 128, 8), (128, 64, 2), (64, 32, 2))    # ConvTranspose1d (Cin, Cout, stride), k = 2 * stride


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


class MelGANVocoder(NeuralVocoder):
    """seungwonpark/melgan's `Generator(mel_channel=80)` on the H100 kernels.

    `forward(mels [B, Lmax, 80], olens [B])` -> (audio [B, Lmax * 256] fp32, alens = olens * 256).  Utterance b is the
    generator applied to mels[b, :olens[b]] followed by 10 frames of -11.5129, every reflection pad at its own edges,
    trimmed to olens[b] * 256 samples; it is bit-identical to a B = 1 call on its own frames whatever else is in the batch,
    audio past alens[b] is 0, and mel frames past olens[b] are never read.  `inference(mel [1, 80, T])` -> int16 [T * 256]
    is the hub object's method.  math_mode: "3xf16" (default, fp32-class), "f16", "tf32" or "fp32" for the GEMMs.  One
    host read per call (the device-side length and range checks)."""

    _NAME, _TAIL = "melgan", 10

    def __init__(self, math_mode: str = "3xf16"):
        super().__init__(math_mode)
        self.mel_channel = N_MELS
        self.generator = _generator()
        self._layers = [m for m in self.modules() if isinstance(m, _WNConv)]      # state_dict order, 42 convolutions

    # ---- checkpoints ----------------------------------------------------------------------------------------------
    @classmethod
    def from_checkpoint(cls, path_or_dict, math_mode: str = "3xf16") -> "MelGANVocoder":
        """seungwonpark/melgan's checkpoint (a dict with "model_g") or a bare generator state dict, given as a file path
        or as the loaded dict.  Either may hold `weight_g` / `weight_v` keys or plain `weight` keys (after
        `remove_weight_norm`, what the hub object holds); a plain weight w is stored as v = w, g = |w|, which folds back to
        w bit for bit.  A missing, unexpected or wrongly shaped key raises ValueError naming it."""
        sd = read_checkpoint(path_or_dict, "model_g", "a generator state dict")
        voc = cls(math_mode=math_mode)
        voc.load_state_dict(normalise_checkpoint(voc, sd))
        return voc

    def eval(self, inference: bool = False):
        """The hub object's signature.  inference=True removes weight norm there; here the folded weights are what the
        kernels use either way, so the audio is the same and the parameters keep their weight_g / weight_v form."""
        super().eval()
        return self

    # ---- device state ---------------------------------------------------------------------------------------------
    def _create(self):
        h = C.c_void_p()
        _lib.check(_lib.load().fs2_melgan_create(C.byref(h), _lib.MATH_MODES[self.math_mode]), "fs2_melgan_create")
        return h.value

    def _load(self, h, device: torch.device) -> None:
        self._load_layers("fs2_melgan_load", h, device)

    def _rows(self, B: int, L: int):
        """fs2_melgan's largest buffer: B * (Lmax + 10) * 256 sample rows."""
        return B * (L + self._TAIL) * HOP, f"B * (Lmax + {self._TAIL}) * {HOP}", "sample"

    def _chain(self):
        """The upsampling strides; a ResStack reads 1 + 3 + 9 rows on each side; the first conv's producer reads mel frames
        for every tap, so level 0 has no wrong rows."""
        return [s for _, _, s in _STAGES], 1 + 3 + 9, 0

    # ---- synthesis ------------------------------------------------------------------------------------------------
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
