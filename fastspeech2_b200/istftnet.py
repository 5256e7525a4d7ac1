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

import torch

from ._kernel_module import HOP, _WNConv
from . import _lib, hifigan

MAX_N_FFT = 16                   # the head kernel's shared memory holds conv_post's outputs for n_fft up to this

# iSTFTNet's published config_v1.json (C8C8I; the fields the generator uses)
CONFIGS = {
    "v1": dict(hifigan.CONFIGS["v1"], upsample_rates=[8, 8], upsample_kernel_sizes=[16, 16], gen_istft_n_fft=16,
               gen_istft_hop_size=4),
}


def load_config(config) -> dict:
    """An iSTFTNet config as a dict of the fields the generator uses: from "v1", a dict (e.g. a loaded config.json) or the
    path of a config.json.  A config without gen_istft_n_fft / gen_istft_hop_size (a hifi-gan config) is refused, naming
    the field.  Only its form is checked here; `check_config` checks what this library runs."""
    return hifigan.load_config(config, CONFIGS, f"one of {sorted(CONFIGS)}", "an iSTFTNet", own=("gen_istft_n_fft", "gen_istft_hop_size"),
                               own_note=" (a hifi-gan config is not an iSTFTNet one)")


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


class ISTFTNetVocoder(hifigan._Generator):
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

    def head_reach(self) -> int:
        """Last-level rows the head reads on each side of its samples' rows: frame f reads rows f - 4 .. f + 2 (conv_post's
        taps and the reflected row) and rows [r0, r1) of samples need frames [r0 - e, r1 + e], e = (n_fft / 2 - 1) // hop."""
        return 4 + (self.config["gen_istft_n_fft"] // 2 - 1) // self.config["gen_istft_hop_size"]

    def _post_reach(self) -> int:
        return self.head_reach()

    def flops_per_frame(self) -> int:
        """Multiply-adds x 2 per mel frame of the generator's convolutions, conv_post's n_fft + 2 outputs included (the
        inverse DFT and overlap-add are not counted)."""
        cfg = self.config
        return super().flops_per_frame() + 2 * HOP // cfg["gen_istft_hop_size"] * \
            (cfg["upsample_initial_channel"] // 2 ** len(cfg["upsample_rates"])) * 7 * (cfg["gen_istft_n_fft"] + 1)

    # ---- device state ---------------------------------------------------------------------------------------------
    def _c_config(self) -> _lib.ISTFTNetConfig:
        c = _lib.ISTFTNetConfig()
        c.gen = hifigan.c_config(self.config)
        c.istft_n_fft = self.config["gen_istft_n_fft"]
        c.istft_hop = self.config["gen_istft_hop_size"]
        return c

    def _load(self, h, device: torch.device) -> None:
        self._load_layers("fs2_istftnet_load", h, device)

    def _rows(self, B: int, L: int):
        """fs2_istftnet's largest GEMM: B * Lmax * (256 / gen_istft_hop_size) last-level rows."""
        up = HOP // self.config["gen_istft_hop_size"]
        return B * L * up, f"B * Lmax * {up}", "row"

