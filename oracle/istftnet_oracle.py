"""CPU oracle of the iSTFTNet vocoder: rishikksh20/iSTFTNet-pytorch's `Generator(h)` restated in torch from the published
architecture (the reference has no iSTFTNet source).  hifi-gan's generator (oracle/hifigan_oracle.py's resblocks) up to
its last MRF, then the head: lrelu(x, 0.01), ReflectionPad1d((1, 0)), conv_post to n_fft + 2 channels, exp of the first
n_fft / 2 + 1 as the magnitude and sin of the rest as the phase, and torch.istft with a periodic Hann window of n_fft
(center=True, onesided, not normalised).  No tanh.  Weight-normalised convolutions, so its state_dict carries the
`g_XXXXXXXX` checkpoints' `weight_g` / `weight_v` keys; `remove_weight_norm()` gives plain `weight` keys.

The key names and the layer layout follow the published code; they have not been checked against a real checkpoint file.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.hifigan_oracle import LRELU_SLOPE, ResBlock1, ResBlock2, _wn

HOP = 256


class Generator(nn.Module):
    """h: a dict with hifi-gan's config fields and gen_istft_n_fft, gen_istft_hop_size."""

    def __init__(self, h: dict, num_mels: int = 80):
        super().__init__()
        self.num_kernels = len(h["resblock_kernel_sizes"])
        self.num_upsamples = len(h["upsample_rates"])
        self.n_fft, self.hop = h["gen_istft_n_fft"], h["gen_istft_hop_size"]
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
        self.reflection_pad = nn.ReflectionPad1d((1, 0))
        self.conv_post = _wn(nn.Conv1d(c0 // 2 ** len(self.ups), self.n_fft + 2, 7, 1, padding=3))

    def body(self, x):
        """mel [B, 80, L] -> the last MRF's output [B, C_U, L * prod(rates)]."""
        x = self.conv_pre(x)
        for i in range(self.num_upsamples):
            x = self.ups[i](F.leaky_relu(x, LRELU_SLOPE))
            xs = None
            for j in range(self.num_kernels):
                r = self.resblocks[i * self.num_kernels + j](x)
                xs = r if xs is None else xs + r
            x = xs / self.num_kernels
        return x

    def post(self, x):
        """conv_post's output [B, n_fft + 2, T + 1] on the last MRF's output x [B, C_U, T]."""
        return self.conv_post(self.reflection_pad(F.leaky_relu(x)))

    def pre_head(self, mel):
        """conv_post's output on mel [B, 80, L]: [B, n_fft + 2, L * prod(rates) + 1]."""
        return self.post(self.body(mel))

    def head(self, x):
        """The last MRF's output [B, C_U, T] -> audio [B, hop * T]."""
        y = self.post(x)
        M = self.n_fft // 2 + 1
        spec, phase = torch.exp(y[:, :M]), torch.sin(y[:, M:])
        window = torch.hann_window(self.n_fft, periodic=True, dtype=x.dtype, device=x.device)
        return torch.istft(spec * torch.exp(1j * phase), self.n_fft, hop_length=self.hop, win_length=self.n_fft, window=window)

    def forward(self, x):
        """mel [B, 80, L] -> audio [B, 1, L * 256]."""
        return self.head(self.body(x))[:, None]

    def remove_weight_norm(self):
        for m in self.modules():
            if hasattr(m, "weight_g"):
                nn.utils.remove_weight_norm(m)


def batched(gen: Generator, mels: torch.Tensor, olens, pre_head: bool = False) -> torch.Tensor:
    """The batched contract, one utterance at a time: mels [B, Lmax, 80], olens [B] -> audio [B, Lmax * 256], each utterance
    the generator on its own frames alone, zero past olens[b] * 256.  pre_head: conv_post's output instead, [B, n_fft + 2,
    Lmax * 256 / hop + 1], zero past column olens[b] * 256 / hop."""
    B, L, _ = mels.shape
    up = HOP // gen.hop
    if pre_head:
        out = torch.zeros(B, gen.n_fft + 2, L * up + 1, dtype=mels.dtype, device=mels.device)
    else:
        out = torch.zeros(B, L * HOP, dtype=mels.dtype, device=mels.device)
    for b, n in enumerate(int(v) for v in olens):
        m = mels[b, :n].T[None]
        if pre_head:
            out[b, :, : n * up + 1] = gen.pre_head(m)[0]
        else:
            out[b, : n * HOP] = gen(m)[0, 0]
    return out
