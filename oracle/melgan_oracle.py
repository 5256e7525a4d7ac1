"""CPU oracle of the MelGAN vocoder: seungwonpark/melgan's `Generator(mel_channel=80)` restated in torch from the
published architecture (the reference loads it with `torch.hub.load("seungwonpark/melgan", "melgan")`, inference.py:180-193,
and keeps no source of it).  Weight-normalised convolutions (`torch.nn.utils.weight_norm`, dim 0), so its state_dict
carries the checkpoint's `weight_g` / `weight_v` keys; `remove_weight_norm()` gives the plain `weight` keys the hub object
holds after `eval(inference=True)`.

The key names and the layer layout follow the published code; they have not been checked against a real checkpoint file.
"""
from __future__ import annotations

import warnings

import torch
import torch.nn as nn

MAX_WAV_VALUE = 32768.0
HOP = 256
TAIL_FRAMES = 10
TAIL_VALUE = -11.5129


def _wn(module):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")          # torch.nn.utils.weight_norm is deprecated in favour of parametrizations
        return nn.utils.weight_norm(module)


class ResStack(nn.Module):
    def __init__(self, channel: int):
        super().__init__()
        self.blocks = nn.ModuleList([nn.Sequential(
            nn.LeakyReLU(0.2), nn.ReflectionPad1d(3 ** i),
            _wn(nn.Conv1d(channel, channel, kernel_size=3, dilation=3 ** i)),
            nn.LeakyReLU(0.2), _wn(nn.Conv1d(channel, channel, kernel_size=1))) for i in range(3)])
        self.shortcuts = nn.ModuleList([_wn(nn.Conv1d(channel, channel, kernel_size=1)) for _ in range(3)])

    def forward(self, x):
        for block, shortcut in zip(self.blocks, self.shortcuts):
            x = shortcut(x) + block(x)
        return x


class Generator(nn.Module):
    def __init__(self, mel_channel: int = 80):
        super().__init__()
        self.mel_channel = mel_channel
        self.generator = nn.Sequential(
            nn.ReflectionPad1d(3), _wn(nn.Conv1d(mel_channel, 512, kernel_size=7)),
            nn.LeakyReLU(0.2), _wn(nn.ConvTranspose1d(512, 256, kernel_size=16, stride=8, padding=4)), ResStack(256),
            nn.LeakyReLU(0.2), _wn(nn.ConvTranspose1d(256, 128, kernel_size=16, stride=8, padding=4)), ResStack(128),
            nn.LeakyReLU(0.2), _wn(nn.ConvTranspose1d(128, 64, kernel_size=4, stride=2, padding=1)), ResStack(64),
            nn.LeakyReLU(0.2), _wn(nn.ConvTranspose1d(64, 32, kernel_size=4, stride=2, padding=1)), ResStack(32),
            nn.LeakyReLU(0.2), nn.ReflectionPad1d(3), _wn(nn.Conv1d(32, 1, kernel_size=7)), nn.Tanh())

    def forward(self, mel):
        return self.generator((mel + 5.0) / 5.0)

    def eval(self, inference: bool = False):
        super().eval()
        if inference:
            self.remove_weight_norm()
        return self

    def remove_weight_norm(self):
        for m in self.modules():
            if hasattr(m, "weight_g"):
                nn.utils.remove_weight_norm(m)

    def inference(self, mel):
        """[1, 80, T] -> int16 [T * 256]: 10 tail frames of -11.5129, forward, trim, * 32768, clamp, truncate."""
        zero = torch.full((1, self.mel_channel, TAIL_FRAMES), TAIL_VALUE).to(mel.device)
        mel = torch.cat((mel, zero), dim=2)
        audio = self.forward(mel).squeeze()
        audio = audio[: -(HOP * TAIL_FRAMES)]
        audio = MAX_WAV_VALUE * audio
        audio = audio.clamp(min=-MAX_WAV_VALUE, max=MAX_WAV_VALUE - 1)
        return audio.short()


def batched(gen: Generator, mels: torch.Tensor, olens) -> torch.Tensor:
    """The batched contract, one utterance at a time: mels [B, Lmax, 80], olens [B] -> fp32 audio [B, Lmax * 256], each
    utterance the generator on its own frames plus the tail frames, trimmed to olens[b] * 256, zero past it."""
    B, L, _ = mels.shape
    out = torch.zeros(B, L * HOP, dtype=mels.dtype)
    for b, n in enumerate(int(v) for v in olens):
        m = mels[b, :n].T[None]
        m = torch.cat((m, torch.full((1, m.shape[1], TAIL_FRAMES), TAIL_VALUE, dtype=m.dtype)), dim=2)
        out[b, : n * HOP] = gen(m)[0, 0, : n * HOP]
    return out
