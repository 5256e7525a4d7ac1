"""CPU oracle of the WaveGlow vocoder: DeepLearningExamples' `WaveGlow` (PyTorch/SpeechSynthesis/Tacotron2/waveglow/
model.py) restated in torch from the published architecture, as the hub entry `nvidia_waveglow` builds it: n_mel_channels
80, n_flows 12, n_group 8, n_early_every 4, n_early_size 2, WN with 8 layers of kernel 3 and n_channels C.  The reference
loads it with `torch.hub.load('nvidia/DeepLearningExamples:torchhub', 'nvidia_waveglow')` (demo_fastspeech2.ipynb, its
"Waveglow" section) and keeps no source of it.

Both directions: `forward(spect, audio)` (audio -> z, the training direction) and `infer(spect, sigma, z=None)`.  WN's
conditioning is DeepLearningExamples' per-layer `cond_layers.{i}` (NVIDIA/waveglow's single `cond_layer` is another
layout).  start, in_layers, cond_layers and res_skip_layers are weight-normalised (`torch.nn.utils.weight_norm`, dim 0),
so the state dict carries `weight_g` / `weight_v` keys; `remove_weightnorm(model)` gives the plain `weight` keys.

The key names and the layer layout follow the published code; they have not been checked against a real checkpoint file,
and neither has which n_channels (256 or 512) NVIDIA's published checkpoint uses.
"""
from __future__ import annotations

import warnings

import torch
import torch.nn as nn
import torch.nn.functional as F

N_MELS = 80
HOP = 256
N_FLOWS, N_GROUP, N_EARLY_EVERY, N_EARLY_SIZE = 12, 8, 4, 2
N_LAYERS, KERNEL_SIZE = 8, 3


def _wn(module):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")          # torch.nn.utils.weight_norm is deprecated in favour of parametrizations
        return nn.utils.weight_norm(module, name="weight")


def flow_channels(k: int) -> int:
    """Audio channels flow k works on: 8, 8, 8, 8, 6, 6, 6, 6, 4, 4, 4, 4."""
    return N_GROUP - N_EARLY_SIZE * (k // N_EARLY_EVERY)


class Invertible1x1Conv(nn.Module):
    def __init__(self, c: int):
        super().__init__()
        self.conv = nn.Conv1d(c, c, kernel_size=1, stride=1, padding=0, bias=False)
        W = torch.linalg.qr(torch.randn(c, c))[0]
        if torch.det(W) < 0:
            W[:, 0] = -1 * W[:, 0]
        self.conv.weight.data = W.view(c, c, 1).contiguous()

    def forward(self, z):
        return self.conv(z)

    def infer(self, z):
        W = self.conv.weight.squeeze(2)
        # DeepLearningExamples inverts in fp32 (W.float().inverse()); a float64 oracle inverts in float64
        W_inverse = (W.inverse() if W.dtype == torch.float64 else W.float().inverse()).to(z.dtype)
        return F.conv1d(z, W_inverse[..., None])


class WN(nn.Module):
    def __init__(self, n_in_channels: int, n_mel_channels: int, n_layers: int, n_channels: int, kernel_size: int):
        super().__init__()
        self.n_layers = n_layers
        self.n_channels = n_channels
        self.in_layers = nn.ModuleList()
        self.res_skip_layers = nn.ModuleList()
        self.cond_layers = nn.ModuleList()
        self.start = _wn(nn.Conv1d(n_in_channels, n_channels, 1))
        end = nn.Conv1d(n_channels, 2 * n_in_channels, 1)      # zero-initialised: every coupling starts as the identity
        end.weight.data.zero_()
        end.bias.data.zero_()
        self.end = end
        for i in range(n_layers):
            dilation = 2 ** i
            padding = (kernel_size * dilation - dilation) // 2
            self.in_layers.append(_wn(nn.Conv1d(n_channels, 2 * n_channels, kernel_size, dilation=dilation, padding=padding)))
            self.cond_layers.append(_wn(nn.Conv1d(n_mel_channels, 2 * n_channels, 1)))
            res_skip_channels = 2 * n_channels if i < n_layers - 1 else n_channels
            self.res_skip_layers.append(_wn(nn.Conv1d(n_channels, res_skip_channels, 1)))

    def forward(self, audio, spect):
        audio = self.start(audio)
        C = self.n_channels
        output = None
        for i in range(self.n_layers):
            in_act = self.in_layers[i](audio) + self.cond_layers[i](spect)
            acts = torch.tanh(in_act[:, :C]) * torch.sigmoid(in_act[:, C:])
            res_skip_acts = self.res_skip_layers[i](acts)
            if i < self.n_layers - 1:
                audio = res_skip_acts[:, :C] + audio
                skip_acts = res_skip_acts[:, C:]
            else:
                skip_acts = res_skip_acts
            output = skip_acts if output is None else skip_acts + output
        return self.end(output)


class WaveGlow(nn.Module):
    def __init__(self, n_channels: int = 512, n_mel_channels: int = N_MELS):
        super().__init__()
        self.upsample = nn.ConvTranspose1d(n_mel_channels, n_mel_channels, 1024, stride=256)
        self.n_flows, self.n_group = N_FLOWS, N_GROUP
        self.n_early_every, self.n_early_size = N_EARLY_EVERY, N_EARLY_SIZE
        self.WN = nn.ModuleList()
        self.convinv = nn.ModuleList()
        n_half = N_GROUP // 2
        n_remaining = N_GROUP
        for k in range(N_FLOWS):
            if k % N_EARLY_EVERY == 0 and k > 0:
                n_half -= N_EARLY_SIZE // 2
                n_remaining -= N_EARLY_SIZE
            self.convinv.append(Invertible1x1Conv(n_remaining))
            self.WN.append(WN(n_half, n_mel_channels * N_GROUP, N_LAYERS, n_channels, KERNEL_SIZE))
        self.n_remaining_channels = n_remaining

    def _cond(self, spect, n_steps):
        """upsample, trim to n_steps * 8 samples, group: [B, 80, T] -> [B, 640, n_steps], channel c * 8 + g."""
        spect = self.upsample(spect)[:, :, : n_steps * self.n_group]
        spect = spect.unfold(2, self.n_group, self.n_group).permute(0, 2, 1, 3)
        return spect.contiguous().view(spect.size(0), spect.size(1), -1).permute(0, 2, 1)

    def forward(self, spect, audio):
        """(mel [B, 80, T], audio [B, T * 256]) -> z [B, 8, T * 32]: channels 0-1 the early output of flow 4, 2-3 that of
        flow 8, 4-7 the last four (DeepLearningExamples returns the log-determinant terms too; they are not needed here)."""
        spect = self._cond(spect, audio.size(1) // self.n_group)
        audio = audio.unfold(1, self.n_group, self.n_group).permute(0, 2, 1)
        out = []
        for k in range(self.n_flows):
            if k % self.n_early_every == 0 and k > 0:
                out.append(audio[:, : self.n_early_size])
                audio = audio[:, self.n_early_size:]
            audio = self.convinv[k](audio)
            n_half = audio.size(1) // 2
            audio_0, audio_1 = audio[:, :n_half], audio[:, n_half:]
            output = self.WN[k](audio_0, spect)
            log_s, b = output[:, n_half:], output[:, :n_half]
            audio = torch.cat([audio_0, torch.exp(log_s) * audio_1 + b], 1)
        out.append(audio)
        return torch.cat(out, 1)

    def infer(self, spect, sigma: float = 1.0, z=None):
        """mel [B, 80, T] -> audio [B, T * 256].  z [B, 8, T * 32] (optional) replaces the three standard-normal draws, in
        forward's layout; without it they come from torch.randn as in DeepLearningExamples."""
        spect = self.upsample(spect)
        time_cutoff = self.upsample.kernel_size[0] - self.upsample.stride[0]
        spect = spect[:, :, :-time_cutoff]
        spect = spect.unfold(2, self.n_group, self.n_group).permute(0, 2, 1, 3)
        spect = spect.contiguous().view(spect.size(0), spect.size(1), -1).permute(0, 2, 1)
        B, T = spect.size(0), spect.size(2)

        def draw(lo, hi):
            if z is not None:
                return z[:, lo:hi].to(spect.dtype)
            return torch.randn(B, hi - lo, T, device=spect.device).to(spect.dtype)

        audio = sigma * draw(N_GROUP - self.n_remaining_channels, N_GROUP)
        for k in reversed(range(self.n_flows)):
            n_half = audio.size(1) // 2
            audio_0, audio_1 = audio[:, :n_half], audio[:, n_half:]
            output = self.WN[k](audio_0, spect)
            s, b = output[:, n_half:], output[:, :n_half]
            audio_1 = (audio_1 - b) / torch.exp(s)
            audio = self.convinv[k].infer(torch.cat([audio_0, audio_1], 1))
            if k % self.n_early_every == 0 and k > 0:
                lo = (k // self.n_early_every - 1) * self.n_early_size
                audio = torch.cat((sigma * draw(lo, lo + self.n_early_size), audio), 1)
        return audio.permute(0, 2, 1).contiguous().view(audio.size(0), -1)

    @staticmethod
    def remove_weightnorm(model):
        for wn in model.WN:
            for m in [wn.start, *wn.in_layers, *wn.cond_layers, *wn.res_skip_layers]:
                nn.utils.remove_weight_norm(m)
        return model


def batched(model: WaveGlow, mels: torch.Tensor, olens, z: torch.Tensor, sigma: float = 1.0) -> torch.Tensor:
    """The batched contract, one utterance at a time: mels [B, Lmax, 80], olens [B], z [B, 8, Lmax * 32] -> audio
    [B, Lmax * 256], utterance b `infer` on its own frames with z[b, :, :olens[b] * 32], zero past olens[b] * 256."""
    B, L, _ = mels.shape
    out = torch.zeros(B, L * HOP, dtype=mels.dtype, device=mels.device)
    for b, n in enumerate(int(v) for v in olens):
        out[b, : n * HOP] = model.infer(mels[b, :n].T[None], sigma, z[b: b + 1, :, : n * HOP // N_GROUP])[0]
    return out
