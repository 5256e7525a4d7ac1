"""CPU oracle of the HiFi-GAN vocoder: jik876/hifi-gan's `Generator(h)` restated in torch from the published architecture
(the reference has no HiFi-GAN source).  Weight-normalised convolutions (`torch.nn.utils.weight_norm`, dim 0), so its
state_dict carries the `g_XXXXXXXX` checkpoints' `weight_g` / `weight_v` keys; `remove_weight_norm()` gives plain `weight`
keys.

The key names and the layer layout follow the published code; they have not been checked against a real checkpoint file.
"""
from __future__ import annotations

import warnings

import torch
import torch.nn as nn
import torch.nn.functional as F

LRELU_SLOPE = 0.1
HOP = 256


def _wn(module):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")          # torch.nn.utils.weight_norm is deprecated in favour of parametrizations
        return nn.utils.weight_norm(module)


def get_padding(kernel_size: int, dilation: int = 1) -> int:
    return (kernel_size * dilation - dilation) // 2


class ResBlock1(nn.Module):
    def __init__(self, channels: int, kernel_size: int = 3, dilation=(1, 3, 5)):
        super().__init__()
        self.convs1 = nn.ModuleList([_wn(nn.Conv1d(channels, channels, kernel_size, 1, dilation=d, padding=get_padding(kernel_size, d)))
                                     for d in dilation[:3]])
        self.convs2 = nn.ModuleList([_wn(nn.Conv1d(channels, channels, kernel_size, 1, dilation=1, padding=get_padding(kernel_size, 1)))
                                     for _ in range(3)])

    def forward(self, x):
        for c1, c2 in zip(self.convs1, self.convs2):
            xt = c2(F.leaky_relu(c1(F.leaky_relu(x, LRELU_SLOPE)), LRELU_SLOPE))
            x = xt + x
        return x


class ResBlock2(nn.Module):
    def __init__(self, channels: int, kernel_size: int = 3, dilation=(1, 3)):
        super().__init__()
        self.convs = nn.ModuleList([_wn(nn.Conv1d(channels, channels, kernel_size, 1, dilation=d, padding=get_padding(kernel_size, d)))
                                    for d in dilation[:2]])

    def forward(self, x):
        for c in self.convs:
            x = c(F.leaky_relu(x, LRELU_SLOPE)) + x
        return x


class Generator(nn.Module):
    """h: a dict with hifi-gan's config fields (resblock, upsample_rates, upsample_kernel_sizes, upsample_initial_channel,
    resblock_kernel_sizes, resblock_dilation_sizes)."""

    def __init__(self, h: dict, num_mels: int = 80):
        super().__init__()
        self.num_kernels = len(h["resblock_kernel_sizes"])
        self.num_upsamples = len(h["upsample_rates"])
        c0 = h["upsample_initial_channel"]
        self.conv_pre = _wn(nn.Conv1d(num_mels, c0, 7, 1, padding=3))
        block = ResBlock1 if str(h["resblock"]) == "1" else ResBlock2
        self.ups = nn.ModuleList([_wn(nn.ConvTranspose1d(c0 // 2 ** i, c0 // 2 ** (i + 1), k, u, padding=(k - u) // 2))
                                  for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"]))])
        self.resblocks = nn.ModuleList()
        for i in range(len(self.ups)):
            ch = c0 // 2 ** (i + 1)
            for k, d in zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"]):
                self.resblocks.append(block(ch, k, d))
        self.conv_post = _wn(nn.Conv1d(c0 // 2 ** len(self.ups), 1, 7, 1, padding=3))

    def pre_tanh(self, x):
        """conv_post's output, before the tanh."""
        x = self.conv_pre(x)
        for i in range(self.num_upsamples):
            x = self.ups[i](F.leaky_relu(x, LRELU_SLOPE))
            xs = None
            for j in range(self.num_kernels):
                r = self.resblocks[i * self.num_kernels + j](x)
                xs = r if xs is None else xs + r
            x = xs / self.num_kernels
        return self.conv_post(F.leaky_relu(x))

    def forward(self, x):
        """mel [B, 80, T] -> audio [B, 1, T * 256]."""
        return torch.tanh(self.pre_tanh(x))

    def remove_weight_norm(self):
        for m in self.modules():
            if hasattr(m, "weight_g"):
                nn.utils.remove_weight_norm(m)


def batched(gen: Generator, mels: torch.Tensor, olens, pre_tanh: bool = False) -> torch.Tensor:
    """The batched contract, one utterance at a time: mels [B, Lmax, 80], olens [B] -> audio [B, Lmax * 256], each utterance
    the generator on its own frames alone, zero past olens[b] * 256 (pre_tanh: conv_post's output instead)."""
    B, L, _ = mels.shape
    out = torch.zeros(B, L * HOP, dtype=mels.dtype, device=mels.device)
    for b, n in enumerate(int(v) for v in olens):
        m = mels[b, :n].T[None]
        out[b, : n * HOP] = (gen.pre_tanh(m) if pre_tanh else gen(m))[0, 0]
    return out
