"""CPU oracle of the BigVGAN vocoder: NVIDIA BigVGAN's generator restated in torch from the published architecture (the
reference has no BigVGAN source).  Weight-normalised convolutions (`torch.nn.utils.weight_norm`, dim 0), so its state_dict
carries the generator checkpoints' `weight_g` / `weight_v` keys; `remove_weight_norm()` gives plain `weight` keys.  Every
layer runs in the module's dtype, so `.double()` gives a float64 oracle.

The key names and the layer layout follow the published code; they have not been checked against a real checkpoint file.
"""
from __future__ import annotations

import math
import warnings

import torch
import torch.nn as nn
import torch.nn.functional as F

HOP = 256


def _wn(module):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")          # torch.nn.utils.weight_norm is deprecated in favour of parametrizations
        return nn.utils.weight_norm(module)


def get_padding(kernel_size: int, dilation: int = 1) -> int:
    return (kernel_size * dilation - dilation) // 2


def kaiser_sinc_filter1d(cutoff: float, half_width: float, kernel_size: int, dtype=torch.float32) -> torch.Tensor:
    """A Kaiser-windowed sinc low-pass of kernel_size taps, normalised to unit sum, as [1, 1, kernel_size]: the Kaiser beta
    from the attenuation A = 2.285 (n/2 - 1) pi 4 half_width + 7.95 (Kaiser's formula), taps at half-integer times for an
    even size."""
    half = kernel_size // 2
    A = 2.285 * (half - 1) * math.pi * 4 * half_width + 7.95
    beta = 0.1102 * (A - 8.7) if A > 50.0 else 0.5842 * (A - 21) ** 0.4 + 0.07886 * (A - 21.0) if A >= 21.0 else 0.0
    window = torch.kaiser_window(kernel_size, periodic=False, beta=beta, dtype=dtype)
    t = (torch.arange(-half, half, dtype=dtype) + 0.5) if kernel_size % 2 == 0 else torch.arange(kernel_size, dtype=dtype) - half
    f = 2 * cutoff * window * torch.sinc(2 * cutoff * t)
    return (f / f.sum()).view(1, 1, kernel_size)


class Snake(nn.Module):
    """x + 1 / (alpha + 1e-9) sin^2(alpha x) per channel (SnakeBeta: 1 / (beta + 1e-9)); with logscale the parameters hold
    log alpha and log beta."""

    def __init__(self, channels: int, beta: bool, logscale: bool):
        super().__init__()
        self.logscale = logscale
        init = torch.zeros(channels) if logscale else torch.ones(channels)
        self.alpha = nn.Parameter(init.clone())
        self.beta = nn.Parameter(init.clone()) if beta else None

    def forward(self, x):
        a = self.alpha[None, :, None]
        b = a if self.beta is None else self.beta[None, :, None]
        if self.logscale:
            a, b = torch.exp(a), torch.exp(b)
        return x + 1.0 / (b + 1e-9) * torch.sin(x * a) ** 2


class _Filter(nn.Module):
    def __init__(self):
        super().__init__()
        self.register_buffer("filter", kaiser_sinc_filter1d(0.25, 0.3, 12))


class _Down(nn.Module):
    def __init__(self):
        super().__init__()
        self.lowpass = _Filter()


class Activation1d(nn.Module):
    """Anti-aliased activation, per channel: 2x upsampling (replicate pad 5, 2 conv_transpose1d with the 12-tap filter,
    stride 2, crop 15 on each side), the activation at the doubled rate, then the low-pass (replicate pad 5 left, 6 right,
    12 taps, stride 2)."""

    def __init__(self, act: nn.Module):
        super().__init__()
        self.act = act
        self.upsample = _Filter()
        self.downsample = _Down()

    def forward(self, x):
        C = x.shape[1]
        f_up = self.upsample.filter.to(x.dtype).expand(C, -1, -1)
        f_down = self.downsample.lowpass.filter.to(x.dtype).expand(C, -1, -1)
        u = 2 * F.conv_transpose1d(F.pad(x, (5, 5), mode="replicate"), f_up, stride=2, groups=C)[..., 15:-15]
        s = self.act(u)
        return F.conv1d(F.pad(s, (5, 6), mode="replicate"), f_down, stride=2, groups=C)


class AMPBlock1(nn.Module):
    def __init__(self, channels: int, kernel_size: int, dilation, beta: bool, logscale: bool):
        super().__init__()
        self.convs1 = nn.ModuleList([_wn(nn.Conv1d(channels, channels, kernel_size, 1, dilation=d, padding=get_padding(kernel_size, d)))
                                     for d in dilation[:3]])
        self.convs2 = nn.ModuleList([_wn(nn.Conv1d(channels, channels, kernel_size, 1, dilation=1, padding=get_padding(kernel_size, 1)))
                                     for _ in range(3)])
        self.activations = nn.ModuleList([Activation1d(Snake(channels, beta, logscale)) for _ in range(6)])

    def forward(self, x):
        for c1, c2, a1, a2 in zip(self.convs1, self.convs2, self.activations[0::2], self.activations[1::2]):
            x = c2(a2(c1(a1(x)))) + x
        return x


class AMPBlock2(nn.Module):
    def __init__(self, channels: int, kernel_size: int, dilation, beta: bool, logscale: bool):
        super().__init__()
        self.convs = nn.ModuleList([_wn(nn.Conv1d(channels, channels, kernel_size, 1, dilation=d, padding=get_padding(kernel_size, d)))
                                    for d in dilation[:2]])
        self.activations = nn.ModuleList([Activation1d(Snake(channels, beta, logscale)) for _ in range(2)])

    def forward(self, x):
        for c, a in zip(self.convs, self.activations):
            x = c(a(x)) + x
        return x


class Generator(nn.Module):
    """h: a dict with BigVGAN's config fields (resblock, upsample_rates, upsample_kernel_sizes, upsample_initial_channel,
    resblock_kernel_sizes, resblock_dilation_sizes, activation, snake_logscale, and optionally use_tanh_at_final and
    use_bias_at_final, both true by default)."""

    def __init__(self, h: dict, num_mels: int = 80):
        super().__init__()
        self.num_kernels = len(h["resblock_kernel_sizes"])
        self.num_upsamples = len(h["upsample_rates"])
        beta, logscale = h["activation"] == "snakebeta", bool(h["snake_logscale"])
        self.use_tanh = bool(h.get("use_tanh_at_final", True))
        c0 = h["upsample_initial_channel"]
        self.conv_pre = _wn(nn.Conv1d(num_mels, c0, 7, 1, padding=3))
        block = AMPBlock1 if str(h["resblock"]) == "1" else AMPBlock2
        self.ups = nn.ModuleList([nn.ModuleList([_wn(nn.ConvTranspose1d(c0 // 2 ** i, c0 // 2 ** (i + 1), k, u, padding=(k - u) // 2))])
                                  for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"]))])
        self.resblocks = nn.ModuleList()
        for i in range(self.num_upsamples):
            ch = c0 // 2 ** (i + 1)
            for k, d in zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"]):
                self.resblocks.append(block(ch, k, d, beta, logscale))
        ch = c0 // 2 ** self.num_upsamples
        self.activation_post = Activation1d(Snake(ch, beta, logscale))
        self.conv_post = _wn(nn.Conv1d(ch, 1, 7, 1, padding=3, bias=bool(h.get("use_bias_at_final", True))))

    def pre_final(self, x):
        """conv_post's output, before the tanh or clamp."""
        x = self.conv_pre(x)
        for i in range(self.num_upsamples):
            x = self.ups[i][0](x)
            xs = None
            for j in range(self.num_kernels):
                r = self.resblocks[i * self.num_kernels + j](x)
                xs = r if xs is None else xs + r
            x = xs / self.num_kernels
        return self.conv_post(self.activation_post(x))

    def forward(self, x):
        """mel [B, 80, T] -> audio [B, 1, T * 256]."""
        y = self.pre_final(x)
        return torch.tanh(y) if self.use_tanh else torch.clamp(y, -1.0, 1.0)

    def remove_weight_norm(self):
        for m in self.modules():
            if hasattr(m, "weight_g"):
                nn.utils.remove_weight_norm(m)


def batched(gen: Generator, mels: torch.Tensor, olens, pre_final: bool = False) -> torch.Tensor:
    """The batched contract, one utterance at a time: mels [B, Lmax, 80], olens [B] -> audio [B, Lmax * 256], each utterance
    the generator on its own frames alone, zero past olens[b] * 256 (pre_final: conv_post's output instead)."""
    B, L, _ = mels.shape
    out = torch.zeros(B, L * HOP, dtype=mels.dtype, device=mels.device)
    for b, n in enumerate(int(v) for v in olens):
        m = mels[b, :n].T[None]
        out[b, : n * HOP] = (gen.pre_final(m) if pre_final else gen(m))[0, 0]
    return out
