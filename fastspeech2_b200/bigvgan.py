"""Batched BigVGAN vocoder on the library's kernels (DESIGN.md section 18).

NVIDIA BigVGAN's 22 kHz 80-band generators read this project's mels as they are when they were trained on fmax 8 kHz mels
(22,050 Hz, n_fft 1024, hop 256, 80 bands from 0 to 8,000 Hz, natural log clamped at 1e-5): `bigvgan_22khz_80band`,
`bigvgan_base_22khz_80band` and `bigvgan_v2_22khz_80band_fmax8k_256x`.  `BigVGANVocoder` runs the generator of a BigVGAN
config batched and per utterance on libfs2b200.so (csrc/bigvgan.cu) and loads its `bigvgan_generator.pt` checkpoints
from a local file.

BigVGAN is HiFi-GAN with every LeakyReLU of the residual blocks replaced by an anti-aliased periodic activation,
`Activation1d(Snake / SnakeBeta)` (2x upsampling with a 12-tap Kaiser-windowed sinc, the activation at the doubled rate,
low-pass and 2x downsampling), no activation before the upsamplings, and an anti-aliased activation before conv_post.  The
module's parameters and buffers carry the checkpoint's keys (`conv_pre.*`, `ups.{i}.0.*`, `resblocks.{j}.convs1.{m}.*` /
`convs2.{m}.*` or `convs.{m}.*`, `resblocks.{j}.activations.{i}.act.alpha` (`.beta`), `...upsample.filter`,
`...downsample.lowpass.filter`, `activation_post.*`, `conv_post.*`; the lists with shapes of the three named configs are
tests/golden/bigvgan_state_dict_keys.json).  They are written from the published code, not checked against a real
checkpoint file.
"""
from __future__ import annotations

import ctypes as C
import math

import torch
import torch.nn as nn

from . import _lib
from ._kernel_module import HOP, N_MELS, _WNConv  # noqa: F401
from . import hifigan
from .hifigan import _Generator, c_config, check_rates, check_resblocks, check_widths

ACT_REACH = 5                    # Activation1d's reach: output row t reads input rows t - 5 .. t + 5
FILTER_TAPS = 12

_22K = {"resblock": "1", "resblock_kernel_sizes": [3, 7, 11], "resblock_dilation_sizes": [[1, 3, 5], [1, 3, 5], [1, 3, 5]],
        "activation": "snakebeta", "snake_logscale": True, "num_mels": 80}
# BigVGAN's published config.json files (the fields the generator uses)
CONFIGS = {
    "base_22khz_80band": dict(_22K, upsample_rates=[8, 8, 2, 2], upsample_kernel_sizes=[16, 16, 4, 4], upsample_initial_channel=512),
    "22khz_80band": dict(_22K, upsample_rates=[4, 4, 2, 2, 2, 2], upsample_kernel_sizes=[8, 8, 4, 4, 4, 4], upsample_initial_channel=1536),
    "v2_22khz_80band_fmax8k_256x": dict(_22K, upsample_rates=[4, 4, 2, 2, 2, 2], upsample_kernel_sizes=[8, 8, 4, 4, 4, 4],
                                        upsample_initial_channel=1536, use_tanh_at_final=False, use_bias_at_final=False),
}


def load_config(config) -> dict:
    """A BigVGAN config as a dict of the fields the generator uses: from a name of CONFIGS, a dict (e.g. a loaded
    config.json) or the path of a config.json.  Only its form is checked here; `check_config` checks what this library
    runs."""
    return hifigan.load_config(config, CONFIGS, f"one of {sorted(CONFIGS)}", "a BigVGAN", fields=("activation", "snake_logscale"),
                               defaults={"use_tanh_at_final": True, "use_bias_at_final": True})


def check_config(cfg: dict) -> None:
    """Raises ValueError naming the field for a config the kernels do not run: anything HiFi-GAN's check_config refuses
    except the widths (num_mels other than 80, which refuses the 24 kHz and 44 kHz models; the upsample rates and kernel
    sizes; the resblock type, kernel sizes and dilations); a convolution width (upsample_initial_channel / 2^i) that is not
    a multiple of 8 or above 2048; an activation other than "snake" / "snakebeta"; snake_logscale, use_tanh_at_final or
    use_bias_at_final that is not a bool."""
    check_rates(cfg)
    check_widths(cfg, 8)
    check_resblocks(cfg)
    if cfg["activation"] not in ("snake", "snakebeta"):
        raise ValueError(f"config: activation must be \"snake\" or \"snakebeta\" (got {cfg['activation']!r})")
    for k in ("snake_logscale", "use_tanh_at_final", "use_bias_at_final"):
        if not isinstance(cfg[k], bool):
            raise ValueError(f"config: {k} must be true or false (got {cfg[k]!r})")


def kaiser_sinc_filter1d(cutoff: float, half_width: float, kernel_size: int) -> torch.Tensor:
    """The default of the Activation1d filter buffers, [1, 1, kernel_size] fp32: a Kaiser-windowed sinc low-pass normalised
    to unit sum (the Kaiser beta from the attenuation 2.285 (n/2 - 1) pi 4 half_width + 7.95; taps at half-integer times
    for an even size).  A checkpoint's own filters replace it."""
    half = kernel_size // 2
    A = 2.285 * (half - 1) * math.pi * 4 * half_width + 7.95
    beta = 0.1102 * (A - 8.7) if A > 50.0 else 0.5842 * (A - 21) ** 0.4 + 0.07886 * (A - 21.0) if A >= 21.0 else 0.0
    window = torch.kaiser_window(kernel_size, periodic=False, beta=beta)
    t = torch.arange(-half, half) + 0.5 if kernel_size % 2 == 0 else torch.arange(kernel_size) - half
    f = 2 * cutoff * window * torch.sinc(2 * cutoff * t)
    return (f / f.sum()).view(1, 1, kernel_size)


class _Snake(nn.Module):
    def __init__(self, c: int, beta: bool, logscale: bool):
        super().__init__()
        init = torch.zeros(c) if logscale else torch.ones(c)
        self.alpha = nn.Parameter(init.clone())
        self.beta = nn.Parameter(init.clone()) if beta else None


class _Filter(nn.Module):
    def __init__(self):
        super().__init__()
        self.register_buffer("filter", kaiser_sinc_filter1d(0.25, 0.3, FILTER_TAPS))


class _Down(nn.Module):
    def __init__(self):
        super().__init__()
        self.lowpass = _Filter()


class _Activation1d(nn.Module):
    def __init__(self, c: int, cfg: dict):
        super().__init__()
        self.act = _Snake(c, cfg["activation"] == "snakebeta", cfg["snake_logscale"])
        self.upsample = _Filter()
        self.downsample = _Down()


class _AMPBlock(nn.Module):
    def __init__(self, c: int, k: int, cfg: dict):
        super().__init__()
        if cfg["resblock"] == "1":
            self.convs1 = nn.ModuleList([_WNConv(c, c, k) for _ in range(3)])
            self.convs2 = nn.ModuleList([_WNConv(c, c, k) for _ in range(3)])
        else:
            self.convs = nn.ModuleList([_WNConv(c, c, k) for _ in range(2)])
        self.activations = nn.ModuleList([_Activation1d(c, cfg) for _ in range(6 if cfg["resblock"] == "1" else 2)])


def add_layers(module: nn.Module, cfg: dict) -> nn.Module:
    """Registers the generator's parameter holders on module, in BigVGAN's order, so that its state_dict keys are the
    checkpoint's: conv_pre, ups, resblocks, activation_post, conv_post."""
    rates, ks, c0 = cfg["upsample_rates"], cfg["upsample_kernel_sizes"], cfg["upsample_initial_channel"]
    module.conv_pre = _WNConv(N_MELS, c0, 7)
    module.ups = nn.ModuleList([nn.ModuleList([_WNConv(c0 // 2 ** i, c0 // 2 ** (i + 1), k, transposed=True)]) for i, k in enumerate(ks)])
    module.resblocks = nn.ModuleList([_AMPBlock(c0 // 2 ** (i + 1), k, cfg) for i in range(len(rates)) for k in cfg["resblock_kernel_sizes"]])
    module.activation_post = _Activation1d(c0 // 2 ** len(rates), cfg)
    module.conv_post = _WNConv(c0 // 2 ** len(rates), 1, 7, bias=cfg["use_bias_at_final"])
    return module


class BigVGANVocoder(_Generator):
    """NVIDIA BigVGAN's generator on the H100 kernels.

    `forward(mels [B, Lmax, 80], olens [B])` -> (audio [B, Lmax * 256] fp32, alens = olens * 256).  Utterance b is the
    generator applied to mels[b, :olens[b]] alone: every convolution zero-pads and every Activation1d replicate-pads at
    its own edges, no tail frames, no mel normalisation.  It is bit-identical to a B = 1 call on its own frames whatever
    else is in the batch, audio past alens[b] is +0, and mel frames past olens[b] are never read.  config: a name of
    CONFIGS, a dict or a config.json path (`check_config` lists what is refused).  math_mode: "3xf16" (default,
    fp32-class), "f16", "tf32" or "fp32" for the GEMMs.  One host read per call.  `window` / `stream` /
    `forward(chunk_frames=)` give the same audio in windows of frames."""

    _NAME = "bigvgan"
    _ACT_REACH = ACT_REACH
    _ACT_FLOP = 2 * 6 + FILTER_TAPS        # per channel and input row: 2 x 6 taps up, 12 taps down; the Snake itself not counted

    def __init__(self, config="base_22khz_80band", math_mode: str = "3xf16"):
        super().__init__(math_mode)
        cfg = load_config(config)
        check_config(cfg)
        self.config = cfg
        add_layers(self, cfg)
        self._layers = [m for m in self.modules() if isinstance(m, _WNConv)]           # state_dict order
        self._acts = [m for m in self.modules() if isinstance(m, _Activation1d)]      # state_dict order, activation_post last

    # ---- device state ---------------------------------------------------------------------------------------------
    def _fingerprint(self):
        return super()._fingerprint() + tuple((b.data_ptr(), b._version) for b in self.buffers())

    def _c_config(self) -> _lib.BigVGANConfig:
        cfg = self.config
        c = _lib.BigVGANConfig()
        c.gen = c_config(cfg)
        c.activation = _lib.FS2_BIGVGAN_SNAKEBETA if cfg["activation"] == "snakebeta" else _lib.FS2_BIGVGAN_SNAKE
        c.snake_logscale = int(cfg["snake_logscale"])
        c.use_tanh_at_final = int(cfg["use_tanh_at_final"])
        c.use_bias_at_final = int(cfg["use_bias_at_final"])
        return c

    def _load(self, h, device: torch.device) -> None:
        def dev(t):
            return None if t is None else t.detach().float().reshape(-1).to(device).contiguous()
        ws = [dev(m.folded()) for m in self._layers]
        bs = [dev(m.bias) for m in self._layers]
        acts = [dev(t) for a in self._acts for t in (a.act.alpha, a.act.beta, a.upsample.filter, a.downsample.lowpass.filter)]

        def ptrs(ts):
            return (C.c_void_p * len(ts))(*[None if t is None else t.data_ptr() for t in ts])
        _lib.check(_lib.load().fs2_bigvgan_load(h, ptrs(ws), ptrs(bs), ptrs(acts), _lib.stream_ptr(device)), "fs2_bigvgan_load")
