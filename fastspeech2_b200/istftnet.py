"""Batched iSTFTNet vocoder on the library's kernels (DESIGN.md section 19).

rishikksh20/iSTFTNet-pytorch's generators read this project's mels as they are (its mel code is hifi-gan's: 22,050 Hz,
n_fft 1024, hop 256, 80 bands from 0 to 8,000 Hz, natural log clamped at 1e-5).  iSTFTNet is hifi-gan's Generator up to
its last MRF, with the last upsamplings replaced by an inverse STFT: conv_post gives n_fft + 2 channels on a
ReflectionPad1d((1, 0)) of lrelu(x, 0.01); exp of the first n_fft / 2 + 1 is the magnitude, sin of the rest the phase, and
`torch.istft(mag * exp(i phase), n_fft, hop, window=hann(n_fft))` the audio, with no tanh.  `ISTFTNetVocoder` runs it
batched and per utterance on libfs2b200.so (the chain in csrc/hifigan.cu, the head in csrc/istftnet.cu) and loads its
`g_XXXXXXXX` checkpoints from a local file.

The module's parameters carry hifi-gan's keys, with conv_post [n_fft + 2, C_U, 7] (the list with shapes for C8C8I is
tests/golden/istftnet_state_dict_keys.json).  They are written from the published code, not checked against a real
checkpoint file.
"""
from __future__ import annotations

import ctypes as C
import json
import os

import torch

from ._kernel_module import HOP, NeuralVocoder, _WNConv, normalise_checkpoint, read_checkpoint, ups_window_plan
from . import _lib, hifigan

MAX_N_FFT = 16                   # the head kernel's shared memory holds conv_post's outputs for n_fft up to this

# iSTFTNet's published config_v1.json (C8C8I; the fields the generator uses)
CONFIGS = {
    "v1": dict(hifigan.CONFIGS["v1"], upsample_rates=[8, 8], upsample_kernel_sizes=[16, 16], gen_istft_n_fft=16,
               gen_istft_hop_size=4),
}
_ISTFT_FIELDS = ("gen_istft_n_fft", "gen_istft_hop_size")


def load_config(config) -> dict:
    """An iSTFTNet config as a dict of the fields the generator uses: from "v1", a dict (e.g. a loaded config.json) or the
    path of a config.json.  A config without gen_istft_n_fft / gen_istft_hop_size (a hifi-gan config) is refused, naming
    the field.  Only its form is checked here; `check_config` checks what this library runs."""
    if isinstance(config, str) and config.lower() in CONFIGS:
        config = CONFIGS[config.lower()]
    elif isinstance(config, (str, os.PathLike)):
        with open(config) as f:
            config = json.load(f)
    if not isinstance(config, dict):
        raise ValueError(f"config must be one of {sorted(CONFIGS)}, a dict or the path of an iSTFTNet config.json")
    for k in _ISTFT_FIELDS:
        if k not in config:
            raise ValueError(f"config: missing field {k} (a hifi-gan config is not an iSTFTNet one)")
    out = hifigan.load_config(config)
    out.update({k: config[k] for k in _ISTFT_FIELDS})
    return out


def check_config(cfg: dict) -> None:
    """Raises ValueError naming the field for a config the kernels do not run: anything HiFi-GAN's check_config refuses
    except the rates' product, which times gen_istft_hop_size must be the hop 256; gen_istft_n_fft odd, below 2 or above 16;
    gen_istft_hop_size that does not divide it with gen_istft_n_fft / gen_istft_hop_size >= 2 (the window envelope would
    be 0)."""
    n, hop = cfg["gen_istft_n_fft"], cfg["gen_istft_hop_size"]
    hifigan._ints("gen_istft_n_fft", [n])
    hifigan._ints("gen_istft_hop_size", [hop])
    if n < 2 or n % 2:
        raise ValueError(f"config: gen_istft_n_fft must be even and at least 2 (got {n})")
    if n > MAX_N_FFT:
        raise ValueError(f"config: gen_istft_n_fft = {n} is above {MAX_N_FFT}, the most the head kernel holds")
    if hop < 1 or n % hop or n // hop < 2:
        raise ValueError(f"config: gen_istft_hop_size = {hop} must divide gen_istft_n_fft = {n} at least twice "
                         "(the window envelope is 0 otherwise)")
    hifigan.check_rates(cfg, hop)
    hifigan.check_widths(cfg, 32)
    hifigan.check_resblocks(cfg)


class ISTFTNetVocoder(NeuralVocoder):
    """rishikksh20/iSTFTNet-pytorch's `Generator(h)` on the H100 kernels.

    `forward(mels [B, Lmax, 80], olens [B])` -> (audio [B, Lmax * 256] fp32, alens = olens * 256).  Utterance b is the
    generator applied to mels[b, :olens[b]] alone: every convolution zero-pads at its own edges, the reflected row and
    the inverse STFT's frames and envelope are the utterance's own, no tail frames, no mel normalisation.  It is
    bit-identical to a B = 1 call on its own frames whatever else is in the batch, audio past alens[b] is +0, and mel
    frames past olens[b] are never read.  config: "v1", a dict or a config.json path (`check_config` lists what is
    refused).  math_mode: "3xf16" (default, fp32-class), "f16", "tf32" or "fp32" for the GEMMs; the head runs in fp32.
    One host read per call.  `window` / `stream` / `forward(chunk_frames=)` give the same audio in windows of frames."""

    _NAME = "istftnet"

    def __init__(self, config="v1", math_mode: str = "3xf16"):
        super().__init__(math_mode)
        cfg = load_config(config)
        check_config(cfg)
        self.config = cfg
        hifigan.add_layers(self, cfg, cfg["gen_istft_n_fft"] + 2)
        self._layers = [m for m in self.modules() if isinstance(m, _WNConv)]      # state_dict order

    def launches(self) -> int:
        """Kernels one call enqueues, as HiFi-GAN's: 4 + U * (2 + K * G + max(K - 2, 0)), G = 12 (resblock "1") or 4."""
        U, K = len(self.config["upsample_rates"]), len(self.config["resblock_kernel_sizes"])
        G = 12 if self.config["resblock"] == "1" else 4
        return 4 + U * (2 + K * G + max(K - 2, 0))

    def head_reach(self) -> int:
        """Last-level rows the head reads on each side of its samples' rows: frame f reads rows f - 4 .. f + 2 (conv_post's
        taps and the reflected row) and rows [r0, r1) of samples need frames [r0 - e, r1 + e], e = (n_fft / 2 - 1) // hop."""
        return 4 + (self.config["gen_istft_n_fft"] // 2 - 1) // self.config["gen_istft_hop_size"]

    def window_plan(self) -> dict:
        """The window plan of this config, walking back from the audio: the head reads head_reach() last-level rows on each
        side, each MRF R, upsampling s reads `reach[s]` input rows around its core, and conv_pre 3 frames more."""
        return ups_window_plan(*self._chain())

    def _chain(self):
        """HiFi-GAN's chain of this config (rates, R, level-0 margin 3) with the head's reach as the last layer's."""
        rates, R, margin0 = hifigan.HiFiGANVocoder._chain(self)
        return rates, R, margin0, self.head_reach()

    def flops_per_frame(self) -> int:
        """Multiply-adds x 2 per mel frame of the generator's convolutions, conv_post's n_fft + 2 outputs included (the
        inverse DFT and overlap-add are not counted)."""
        cfg = self.config
        return hifigan.HiFiGANVocoder.flops_per_frame(self) + 2 * HOP // cfg["gen_istft_hop_size"] * \
            (cfg["upsample_initial_channel"] // 2 ** len(cfg["upsample_rates"])) * 7 * (cfg["gen_istft_n_fft"] + 1)

    # ---- checkpoints ----------------------------------------------------------------------------------------------
    @classmethod
    def from_checkpoint(cls, path_or_dict, config=None, math_mode: str = "3xf16") -> "ISTFTNetVocoder":
        """An iSTFTNet generator checkpoint (`g_XXXXXXXX`: a dict with "generator") or a bare generator state dict, given
        as a file path or as the loaded dict, with `weight_g` / `weight_v` or plain `weight` keys.  config: as in the
        constructor; None reads config.json beside a checkpoint path.  A missing, unexpected or wrongly shaped key raises
        ValueError naming it."""
        sd = path_or_dict
        if config is None:
            if not isinstance(sd, (str, os.PathLike)):
                raise ValueError("config is required when the checkpoint is given as a dict")
            path = os.path.join(os.path.dirname(os.path.abspath(sd)), "config.json")
            if not os.path.exists(path):
                raise ValueError(f"config is required: no config.json beside {sd}")
            config = path
        voc = cls(config, math_mode=math_mode)
        voc.load_state_dict(normalise_checkpoint(voc, read_checkpoint(sd, "generator", "a generator state dict")))
        return voc

    # ---- device state ---------------------------------------------------------------------------------------------
    def _c_config(self) -> _lib.ISTFTNetConfig:
        c = _lib.ISTFTNetConfig()
        c.gen = hifigan.c_config(self.config)
        c.istft_n_fft = self.config["gen_istft_n_fft"]
        c.istft_hop = self.config["gen_istft_hop_size"]
        return c

    def _create(self):
        h = C.c_void_p()
        cfg = self._c_config()
        _lib.check(_lib.load().fs2_istftnet_create(C.byref(h), _lib.MATH_MODES[self.math_mode], C.byref(cfg)), "fs2_istftnet_create")
        return h.value

    def _load(self, h, device: torch.device) -> None:
        self._load_layers("fs2_istftnet_load", h, device)

    def _rows(self, B: int, L: int):
        """fs2_istftnet's largest GEMM: B * Lmax * (256 / gen_istft_hop_size) last-level rows."""
        up = HOP // self.config["gen_istft_hop_size"]
        return B * L * up, f"B * Lmax * {up}", "row"

