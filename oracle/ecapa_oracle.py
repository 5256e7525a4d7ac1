"""A torch restatement of SpeechBrain's ECAPA-TDNN speaker encoder (`speechbrain/spkrec-ecapa-voxceleb`), written from
SpeechBrain's published code: `Fbank(n_mels=80)`, `InputNormalization(norm_type="sentence", std_norm=False)` and
`ECAPA_TDNN`.  The module tree's state_dict keys are SpeechBrain's (the Conv1d / BatchNorm1d wrappers hold the torch
layer as `.conv` / `.norm`).  `embed` runs one utterance at a time, in the dtype of its input (float64 in the tests): each
convolution is "same" with reflect padding at the utterance's own edges, every mean is over the utterance's own frames.

Neither the keys nor the arithmetic have been checked against a real checkpoint or against SpeechBrain itself (DESIGN.md
section 28)."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

SAMPLE_RATE, N_FFT, HOP, WIN, TOP_DB, AMIN = 16000, 400, 160, 400, 80.0, 1e-10


class _Conv(nn.Module):
    """speechbrain.nnet.CNN.Conv1d: the torch layer under `.conv`; "same" padding with reflect at the edges."""

    def __init__(self, cin, cout, k, d=1):
        super().__init__()
        self.conv = nn.Conv1d(cin, cout, k, dilation=d)
        self.pad = d * (k - 1) // 2

    def forward(self, x):                      # x [C, T] or [B, C, T]
        xb = x if x.dim() == 3 else x[None]
        if self.pad:
            xb = F.pad(xb, (self.pad, self.pad), mode="reflect")
        y = F.conv1d(xb, self.conv.weight.to(x.dtype), self.conv.bias.to(x.dtype), dilation=self.conv.dilation)
        return y if x.dim() == 3 else y[0]


class _BN(nn.Module):
    """speechbrain.nnet.normalization.BatchNorm1d: the torch layer under `.norm`, applied in eval mode."""

    def __init__(self, c):
        super().__init__()
        self.norm = nn.BatchNorm1d(c)

    def forward(self, x):                      # x [C, T], [B, C, T] or [C]
        n = self.norm
        sh = (-1,) + (1,) * min(x.dim() - 1, 1)
        return ((x - n.running_mean.to(x.dtype).reshape(sh)) / torch.sqrt(n.running_var.to(x.dtype).reshape(sh) + n.eps)
                * n.weight.to(x.dtype).reshape(sh) + n.bias.to(x.dtype).reshape(sh))


class TDNNBlock(nn.Module):
    def __init__(self, cin, cout, k, d=1):
        super().__init__()
        self.conv = _Conv(cin, cout, k, d)
        self.norm = _BN(cout)

    def forward(self, x):
        return self.norm(torch.relu(self.conv(x)))


class Res2NetBlock(nn.Module):
    def __init__(self, c, scale, k, d):
        super().__init__()
        self.scale = scale
        self.blocks = nn.ModuleList([TDNNBlock(c // scale, c // scale, k, d) for _ in range(scale - 1)])

    def forward(self, x):
        ys = []
        for i, xi in enumerate(torch.chunk(x, self.scale, dim=-2)):
            y = xi if i == 0 else self.blocks[i - 1](xi) if i == 1 else self.blocks[i - 1](xi + y)
            ys.append(y)
        return torch.cat(ys, -2)


class SEBlock(nn.Module):
    def __init__(self, c, se):
        super().__init__()
        self.conv1 = _Conv(c, se, 1)
        self.conv2 = _Conv(se, c, 1)

    def forward(self, x):
        s = x.mean(-1, keepdim=True)
        return torch.sigmoid(self.conv2(torch.relu(self.conv1(s)))) * x


class SERes2NetBlock(nn.Module):
    def __init__(self, c, scale, se, k, d):
        super().__init__()
        self.tdnn1 = TDNNBlock(c, c, 1)
        self.res2net_block = Res2NetBlock(c, scale, k, d)
        self.tdnn2 = TDNNBlock(c, c, 1)
        self.se_block = SEBlock(c, se)

    def forward(self, x):
        return self.se_block(self.tdnn2(self.res2net_block(self.tdnn1(x)))) + x


def _stats(x, w):
    """SpeechBrain's _compute_statistics over time with weights w [1 or C, T]: mean, sqrt(clamp(var, 1e-12))."""
    mean = (w * x).sum(-1)
    return mean, torch.sqrt((w * (x - mean[..., None]) ** 2).sum(-1).clamp(min=1e-12))


class AttentiveStatisticsPooling(nn.Module):
    def __init__(self, c, att, global_context=True):
        super().__init__()
        self.global_context = global_context
        self.tdnn = TDNNBlock(c * 3 if global_context else c, att, 1)
        self.conv = _Conv(att, c, 1)

    def forward(self, x, fold: bool = False):   # x [C, T] -> [2C], or [B, C, T] -> [B, 2C]
        T = x.shape[-1]
        a = x
        if self.global_context:
            m, s = _stats(x, torch.full((1, T), 1.0 / T, dtype=x.dtype, device=x.device))
            if fold:   # W [h; mu; sigma] = W_h h + (W_mu mu + W_sigma sigma): the library's form
                W = self.tdnn.conv.conv.weight.to(x.dtype)[:, :, 0]
                C = x.shape[0]
                ctx = W[:, C:2 * C] @ m + W[:, 2 * C:] @ s + self.tdnn.conv.conv.bias.to(x.dtype)
                z = W[:, :C] @ x + ctx[:, None]
                a = torch.tanh(self.tdnn.norm(torch.relu(z)))
                return self._pool(x, self.conv(a))
            a = torch.cat([x, m[..., None].expand(*m.shape, T), s[..., None].expand(*s.shape, T)], -2)
        return self._pool(x, self.conv(torch.tanh(self.tdnn(a))))

    @staticmethod
    def _pool(x, logits):
        w = torch.softmax(logits, dim=-1)
        m, s = _stats(x, w)
        return torch.cat([m, s], -1)


class ECAPA_TDNN(nn.Module):
    """SpeechBrain's ECAPA_TDNN(input_size, channels, kernel_sizes, dilations, attention_channels, res2net_scale,
    se_channels, global_context, lin_neurons), eval semantics, one utterance at a time."""

    def __init__(self, input_size=80, channels=(1024, 1024, 1024, 1024, 3072), kernel_sizes=(5, 3, 3, 3, 1),
                 dilations=(1, 2, 3, 4, 1), attention_channels=128, res2net_scale=8, se_channels=128, global_context=True,
                 lin_neurons=192):
        super().__init__()
        self.blocks = nn.ModuleList([TDNNBlock(input_size, channels[0], kernel_sizes[0], dilations[0])])
        for i in range(1, len(channels) - 1):
            self.blocks.append(SERes2NetBlock(channels[i], res2net_scale, se_channels, kernel_sizes[i], dilations[i]))
        self.mfa = TDNNBlock(sum(channels[1:-1]), channels[-1], kernel_sizes[-1], dilations[-1])
        self.asp = AttentiveStatisticsPooling(channels[-1], attention_channels, global_context)
        self.asp_bn = _BN(channels[-1] * 2)
        self.fc = _Conv(channels[-1] * 2, lin_neurons, 1)

    def forward(self, feats, fold: bool = False):  # feats [T, n_mels] -> [D], or [B, T, n_mels] -> [B, D] (padded frames count)
        x = feats.transpose(-1, -2)
        xl = []
        for blk in self.blocks:
            x = blk(x)
            xl.append(x)
        x = self.mfa(torch.cat(xl[1:], -2))
        return self.fc(self.asp_bn(self.asp(x, fold)[..., None]))[..., 0]

    def embed(self, wav, fold: bool = False):
        """One utterance's embedding [D] from its 16 kHz samples [N] (in wav's dtype)."""
        return self(features(wav), fold)


# ---- front end ----------------------------------------------------------------------------------------------------

def mel_filterbank(n_mels=80, n_fft=N_FFT, sr=SAMPLE_RATE, dtype=torch.float64):
    """SpeechBrain's Filterbank matrix [n_fft // 2 + 1, n_mels]: symmetric triangles of half-width `band` (the spacing to
    the lower neighbour), not area-normalised."""
    mel = lambda f: 2595.0 * np.log10(1.0 + f / 700.0)                   # noqa: E731
    m = np.linspace(mel(0.0), mel(sr / 2), n_mels + 2)
    hz = 700.0 * (10.0 ** (m / 2595.0) - 1.0)
    band = (hz[1:] - hz[:-1])[:-1]
    fc = hz[1:-1]
    f = np.linspace(0, sr / 2, n_fft // 2 + 1)
    slope = (f[:, None] - fc[None, :]) / band[None, :]
    return torch.from_numpy(np.maximum(0.0, np.minimum(slope + 1.0, 1.0 - slope))).to(dtype)


def fbank_db(wav):
    """[T, n_mels] log-mel power in dB, T = 1 + N // 160, with the top-db clamp (before the mean normalisation)."""
    win = torch.hamming_window(WIN, periodic=True, dtype=wav.dtype, device=wav.device)
    X = torch.stft(wav, N_FFT, HOP, WIN, window=win, center=True, pad_mode="constant", return_complex=True)
    p = X.real ** 2 + X.imag ** 2                                        # [201, T]
    mel = p.t() @ mel_filterbank(dtype=wav.dtype).to(wav.device)
    db = 10.0 * torch.log10(mel.clamp(min=AMIN))
    return torch.maximum(db, db.max() - TOP_DB)


def features(wav):
    """Fbank + sentence mean normalisation: [T, n_mels]."""
    db = fbank_db(wav)
    return db - db.mean(0, keepdim=True)


def n_frames(n: int) -> int:
    return 1 + n // HOP


def config_of(model: ECAPA_TDNN) -> dict:
    """The constructor arguments the weights' shapes imply (dilations are not stored)."""
    return {"C": model.blocks[1].tdnn1.conv.conv.weight.shape[0]}


def seeded(seed: int = 0, **kw) -> ECAPA_TDNN:
    """An ECAPA_TDNN with seeded random weights: every convolution scaled to keep unit-scale activations once the
    BatchNorm statistics are set (`calibrate`)."""
    g = torch.Generator().manual_seed(seed)
    m = ECAPA_TDNN(**kw)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if p.dim() == 3:
                fan = p.shape[1] * p.shape[2]
                p.copy_(torch.randn(p.shape, generator=g) / math.sqrt(fan))
            elif name.endswith("conv.bias"):
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
            elif name.endswith("norm.weight"):
                p.copy_(1.0 + 0.1 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
    return m


@torch.no_grad()
def calibrate(model: ECAPA_TDNN, wavs) -> None:
    """Sets every BatchNorm's running mean and variance to the statistics of its input over the frames of `wavs` (a list
    of 1-D float64 tensors), in a float64 pass, layer by layer, so that activations stay at unit scale through the depth.
    asp_bn, fed one vector per utterance, gets the mean and variance over the utterances."""
    bns = [m for m in model.modules() if isinstance(m, _BN)]
    for bn in bns:
        n = bn.norm
        n.running_mean.zero_()
        n.running_var.fill_(1.0)
        n.weight.fill_(1.0)
        n.bias.zero_()
    model.double()
    for bn in bns:
        seen = []
        hook = bn.register_forward_pre_hook(lambda mod, inp: seen.append(inp[0].detach()))
        for w in wavs:
            model.embed(w.double())
        hook.remove()
        x = torch.cat([s if s.dim() == 2 else s[:, None] for s in seen], 1)
        bn.norm.running_mean.copy_(x.mean(1))
        bn.norm.running_var.copy_(x.var(1, unbiased=False).clamp(min=1e-6))
    model.float()


def state_dict_shapes(model: nn.Module) -> dict:
    return {k: list(v.shape) for k, v in model.state_dict().items()}
