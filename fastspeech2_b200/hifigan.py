"""Batched HiFi-GAN vocoder on the library's kernels (DESIGN.md section 16).

jik876/hifi-gan's generators read this project's mels as they are: 22,050 Hz, n_fft 1024, hop 256, 80 bands from 0 to
8,000 Hz, natural log clamped at 1e-5.  `HiFiGANVocoder` runs the `Generator` of a hifi-gan config batched and per utterance
on libfs2b200.so (csrc/hifigan.cu) and loads its `g_XXXXXXXX` checkpoints from a local file.

The module's parameters carry the checkpoint's keys (`conv_pre.{bias,weight_g,weight_v}`, `ups.{i}.*`,
`resblocks.{j}.convs1.{m}.*` / `convs2.{m}.*` or `resblocks.{j}.convs.{m}.*`, `conv_post.*`; the lists with shapes for V1,
V2 and V3 are tests/golden/hifigan_state_dict_keys.json).  They are written from the published code, not checked against a
real checkpoint file.
"""
from __future__ import annotations

import ctypes as C
import json
import math
import os

import torch
import torch.nn as nn

from . import _lib
from ._kernel_module import (HOP, MAX_WAV_VALUE, N_MELS, NeuralVocoder, _WNConv, normalise_checkpoint, read_checkpoint,  # noqa: F401
                             ups_window_plan)

# hifi-gan's published config_v1.json, config_v2.json and config_v3.json (the fields the generator uses).  V2's widths
# (128 ... 8) are refused by HiFiGANVocoder; the entry is here for its key list.
CONFIGS = {
    "v1": {"resblock": "1", "upsample_rates": [8, 8, 2, 2], "upsample_kernel_sizes": [16, 16, 4, 4], "upsample_initial_channel": 512,
           "resblock_kernel_sizes": [3, 7, 11], "resblock_dilation_sizes": [[1, 3, 5], [1, 3, 5], [1, 3, 5]], "num_mels": 80},
    "v2": {"resblock": "1", "upsample_rates": [8, 8, 2, 2], "upsample_kernel_sizes": [16, 16, 4, 4], "upsample_initial_channel": 128,
           "resblock_kernel_sizes": [3, 7, 11], "resblock_dilation_sizes": [[1, 3, 5], [1, 3, 5], [1, 3, 5]], "num_mels": 80},
    "v3": {"resblock": "2", "upsample_rates": [8, 8, 4], "upsample_kernel_sizes": [16, 16, 8], "upsample_initial_channel": 256,
           "resblock_kernel_sizes": [3, 5, 7], "resblock_dilation_sizes": [[1, 2], [2, 6], [3, 12]], "num_mels": 80},
}
_FIELDS = ("resblock", "upsample_rates", "upsample_kernel_sizes", "upsample_initial_channel", "resblock_kernel_sizes",
           "resblock_dilation_sizes")


def load_config(config, configs=None, choices: str = "'v1', 'v2', 'v3'", what: str = "a hifi-gan", fields=(), defaults=None,
                own=(), own_note: str = "") -> dict:
    """A hifi-gan config as a dict of the fields the generator uses: from "v1" / "v2" / "v3", a dict (e.g. a loaded
    config.json) or the path of a config.json.  Only its form is checked here; `check_config` checks what this library
    runs.

    BigVGAN's and iSTFTNet's load_config are this one on their own configs (a name of `configs`, refused as "config must
    be <choices>, a dict or the path of <what> config.json"), with more fields: `own`, required before hifi-gan's
    (missing: "config: missing field <k><own_note>"); `fields`, required after them; `defaults`, optional with defaults."""
    configs = CONFIGS if configs is None else configs
    if isinstance(config, str) and config.lower() in configs:
        config = configs[config.lower()]
    elif isinstance(config, (str, os.PathLike)):
        with open(config) as f:
            config = json.load(f)
    if not isinstance(config, dict):
        raise ValueError(f"config must be {choices}, a dict or the path of {what} config.json")
    for k in own:
        if k not in config:
            raise ValueError(f"config: missing field {k}{own_note}")
    for k in _FIELDS + tuple(fields):
        if k not in config:
            raise ValueError(f"config: missing field {k}")
    out = {"resblock": str(config["resblock"]), "upsample_initial_channel": config["upsample_initial_channel"]}
    out.update({k: config[k] for k in fields})
    out.update({k: config.get(k, v) for k, v in (defaults or {}).items()})
    for k in ("upsample_rates", "upsample_kernel_sizes", "resblock_kernel_sizes"):
        out[k] = [v for v in config[k]]
    out["resblock_dilation_sizes"] = [list(d) for d in config["resblock_dilation_sizes"]]
    if "num_mels" in config:
        out["num_mels"] = config["num_mels"]
    out.update({k: config[k] for k in own})
    return out


def _ints(name, values):
    if not all(isinstance(v, int) and not isinstance(v, bool) for v in values):
        raise ValueError(f"config: {name} must hold integers")


def check_config(cfg: dict) -> None:
    """Raises ValueError naming the field for a config the kernels do not run: num_mels other than 80; a resblock type
    other than "1" or "2"; upsample rates that are odd, whose product is not the hop 256, or whose kernel sizes are not
    twice the rate; a convolution width (upsample_initial_channel / 2^i) that is not a multiple of 32 (this refuses V2) or
    above 2048; even resblock kernel sizes; too few dilations per resblock."""
    check_rates(cfg)
    check_widths(cfg, 32)
    check_resblocks(cfg)


def check_rates(cfg: dict, head_hop: int = 1) -> None:
    """check_config's rules before the widths: num_mels, the resblock type, the upsample rates and kernel sizes.
    head_hop: the samples per last-level row of the head (iSTFTNet's gen_istft_hop_size), which the rates' product times
    must give the hop 256."""
    if cfg.get("num_mels", N_MELS) != N_MELS:
        raise ValueError(f"config: num_mels must be {N_MELS} (got {cfg['num_mels']})")
    if cfg["resblock"] not in ("1", "2"):
        raise ValueError(f"config: resblock must be \"1\" or \"2\" (got {cfg['resblock']!r})")
    rates, ks = cfg["upsample_rates"], cfg["upsample_kernel_sizes"]
    _ints("upsample_rates", rates)
    _ints("upsample_kernel_sizes", ks)
    if not 1 <= len(rates) <= _lib.FS2_HIFIGAN_MAX_UPSAMPLES:
        raise ValueError(f"config: upsample_rates must hold 1 to {_lib.FS2_HIFIGAN_MAX_UPSAMPLES} rates")
    if any(u < 2 or u % 2 for u in rates):
        raise ValueError(f"config: upsample_rates must be even (got {rates})")
    if head_hop == 1 and math.prod(rates) != HOP:
        raise ValueError(f"config: the product of upsample_rates must be the hop {HOP} (got {math.prod(rates)})")
    if math.prod(rates) * head_hop != HOP:
        raise ValueError(f"config: the product of upsample_rates times gen_istft_hop_size must be the hop {HOP} "
                         f"(got {math.prod(rates)} * {head_hop})")
    if len(ks) != len(rates) or any(k != 2 * u for k, u in zip(ks, rates)):
        raise ValueError(f"config: upsample_kernel_sizes must be twice the upsample_rates (got {ks} for {rates})")


def check_widths(cfg: dict, multiple: int) -> None:
    """Every convolution width upsample_initial_channel / 2^i a multiple of `multiple`, at most 2048."""
    c0, rates = cfg["upsample_initial_channel"], cfg["upsample_rates"]
    _ints("upsample_initial_channel", [c0])
    widths = [c0 // 2 ** i for i in range(len(rates) + 1)]
    if c0 > 2048 or c0 % 2 ** len(rates) or any(w % multiple or w < multiple for w in widths):
        raise ValueError(f"config: upsample_initial_channel = {c0} gives convolution widths {widths}; every one must be a "
                         f"multiple of {multiple} (and at most 2048)")


def check_resblocks(cfg: dict) -> None:
    """check_config's rules after the widths: the resblock kernel sizes and dilations."""
    kers, dils = cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"]
    _ints("resblock_kernel_sizes", kers)
    if not 1 <= len(kers) <= _lib.FS2_HIFIGAN_MAX_KERNELS or any(k < 1 or k > 31 or k % 2 == 0 for k in kers):
        raise ValueError(f"config: resblock_kernel_sizes must be 1 to {_lib.FS2_HIFIGAN_MAX_KERNELS} odd sizes in [1, 31] (got {kers})")
    need = 3 if cfg["resblock"] == "1" else 2
    if len(dils) != len(kers) or any(len(d) < need for d in dils):
        raise ValueError(f"config: resblock_dilation_sizes must hold {need} dilations for each of the {len(kers)} kernel sizes")
    for d in dils:
        _ints("resblock_dilation_sizes", d)
        if any(v < 1 or v > 1024 for v in d[:need]):
            raise ValueError(f"config: resblock_dilation_sizes must lie in [1, 1024] (got {dils})")


def c_config(cfg: dict) -> _lib.HiFiGANConfig:
    """The fs2_hifigan_config of a checked config."""
    c = _lib.HiFiGANConfig()
    c.resblock = int(cfg["resblock"])
    c.num_upsamples = len(cfg["upsample_rates"])
    for i, (u, k) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"])):
        c.upsample_rates[i], c.upsample_kernel_sizes[i] = u, k
    c.upsample_initial_channel = cfg["upsample_initial_channel"]
    c.num_kernels = len(cfg["resblock_kernel_sizes"])
    c.num_dilations = 3 if c.resblock == 1 else 2
    for j, (k, d) in enumerate(zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"])):
        c.resblock_kernel_sizes[j] = k
        for m in range(c.num_dilations):
            c.resblock_dilation_sizes[j][m] = d[m]
    return c


class _ResBlock1(nn.Module):
    def __init__(self, c: int, k: int):
        super().__init__()
        self.convs1 = nn.ModuleList([_WNConv(c, c, k) for _ in range(3)])
        self.convs2 = nn.ModuleList([_WNConv(c, c, k) for _ in range(3)])


class _ResBlock2(nn.Module):
    def __init__(self, c: int, k: int):
        super().__init__()
        self.convs = nn.ModuleList([_WNConv(c, c, k) for _ in range(2)])


def add_layers(module: nn.Module, cfg: dict, post_channels: int = 1) -> nn.Module:
    """Registers the generator's parameter holders on module, in hifi-gan's order, so that its state_dict keys are the
    checkpoint's: conv_pre, ups, resblocks, conv_post (post_channels outputs: 1, or iSTFTNet's n_fft + 2).  No check of
    the config beyond its shapes (the key lists of configs the kernels refuse, such as V2, come from here too)."""
    rates, ks, c0 = cfg["upsample_rates"], cfg["upsample_kernel_sizes"], cfg["upsample_initial_channel"]
    block = _ResBlock1 if str(cfg["resblock"]) == "1" else _ResBlock2
    module.conv_pre = _WNConv(N_MELS, c0, 7)
    module.ups = nn.ModuleList([_WNConv(c0 // 2 ** i, c0 // 2 ** (i + 1), k, transposed=True) for i, k in enumerate(ks)])
    module.resblocks = nn.ModuleList([block(c0 // 2 ** (i + 1), k) for i in range(len(rates)) for k in cfg["resblock_kernel_sizes"]])
    module.conv_post = _WNConv(c0 // 2 ** len(rates), post_channels, 7)
    return module


class _Generator(NeuralVocoder):
    """What HiFiGANVocoder, BigVGANVocoder and ISTFTNetVocoder share: hifi-gan's generator chain (csrc/hifigan.cu) with
    the activation before its block convolutions reaching _ACT_REACH rows on each side (lrelu: 0) and costing _ACT_FLOP
    multiply-adds per channel and row (lrelu: 0).  A subclass sets self.config and self._layers and provides _c_config()."""

    _ACT_REACH = 0
    _ACT_FLOP = 0

    def launches(self) -> int:
        """Kernels one call enqueues: 4 + U * (2 + K * G + max(K - 2, 0)), G = 12 (resblock "1") or 4 (resblock "2")."""
        U, K = len(self.config["upsample_rates"]), len(self.config["resblock_kernel_sizes"])
        G = 12 if self.config["resblock"] == "1" else 4
        return 4 + U * (2 + K * G + max(K - 2, 0))

    def window_plan(self) -> dict:
        """The window plan of this config (DESIGN.md section 17), walking back from the audio: the head reads its reach
        (conv_post: 3 rows on each side) of the last level, each MRF R = its largest resblock's reach, upsampling s reads
        `reach[s]` input rows around its core, and conv_pre 3 frames more.  -> {"reach": [r_s], "halo": [h_s] (rows of
        level s on each side of its core; h_0 = r_0 + 3 mel frames, h_{s+1} = u_s r_s), "R": R}."""
        return ups_window_plan(*self._chain())

    def _chain(self):
        """The upsample rates; R = the largest resblock's reach, its activations' included (ResBlock1 sum_m ((k-1)/2
        (d_m + 1) + 2 a), ResBlock2 sum_m ((k-1)/2 d_m + a), a = _ACT_REACH); conv_pre's native taps leave its 3 outer rows
        wrong at a window side that is not an utterance edge; the last layer's reach."""
        cfg, a = self.config, self._ACT_REACH
        one = cfg["resblock"] == "1"
        steps = 3 if one else 2
        R = max(sum((k - 1) // 2 * (d + one) + (2 if one else 1) * a for d in dil[:steps])
                for k, dil in zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"]))
        return cfg["upsample_rates"], R, 3, self._post_reach()

    def _post_reach(self) -> int:
        """Last-level rows the head reads on each side: conv_post's 3, through its activation's reach."""
        return 3 + self._ACT_REACH

    def flops_per_frame(self) -> int:
        """FLOP per mel frame: multiply-adds x 2 of the generator's convolutions (the transposed ones counted as torch runs
        them: Cin * Cout * k per input row) and of its activations (_ACT_FLOP per channel and input row)."""
        cfg = self.config
        c0, f = cfg["upsample_initial_channel"], 0
        f += N_MELS * c0 * 7
        up = 1
        convs = 6 if cfg["resblock"] == "1" else 2
        act = self._ACT_FLOP
        for i, (u, k) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"])):
            cin, cout = c0 // 2 ** i, c0 // 2 ** (i + 1)
            f += up * cin * cout * k
            up *= u
            f += up * sum(convs * cout * cout * kk + convs * cout * act for kk in cfg["resblock_kernel_sizes"])
        f += up * (c0 // 2 ** len(cfg["upsample_rates"])) * (act + 7)
        return 2 * f

    # ---- checkpoints ----------------------------------------------------------------------------------------------
    @classmethod
    def from_checkpoint(cls, path_or_dict, config=None, math_mode: str = "3xf16"):
        """A generator checkpoint (hifi-gan's and iSTFTNet's `g_XXXXXXXX`, BigVGAN's `bigvgan_generator.pt`: a dict with
        "generator") or a bare generator state dict, given as a file path or as the loaded dict.  Either may hold
        `weight_g` / `weight_v` keys or plain `weight` keys (after `remove_weight_norm`); BigVGAN's filters are the
        checkpoint's own.  config: as in the constructor; None reads config.json beside a checkpoint path, as hifi-gan's
        inference.py does (the dilations cannot be read from the weights).  A missing, unexpected or wrongly shaped key
        raises ValueError naming it."""
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
    def _create(self):
        h = C.c_void_p()
        cfg = self._c_config()
        name = f"fs2_{self._NAME}_create"
        _lib.check(getattr(_lib.load(), name)(C.byref(h), _lib.MATH_MODES[self.math_mode], C.byref(cfg)), name)
        return h.value

    def _rows(self, B: int, L: int):
        """fs2_<_NAME>'s largest buffer: B * Lmax * 256 sample rows."""
        return B * L * HOP, f"B * Lmax * {HOP}", "sample"


class HiFiGANVocoder(_Generator):
    """jik876/hifi-gan's `Generator(h)` on the H100 kernels.

    `forward(mels [B, Lmax, 80], olens [B])` -> (audio [B, Lmax * 256] fp32, alens = olens * 256).  Utterance b is the
    generator applied to mels[b, :olens[b]] alone: every convolution zero-pads at its own edges, no tail frames, no mel
    normalisation.  It is bit-identical to a B = 1 call on its own frames whatever else is in the batch, audio past
    alens[b] is +0, and mel frames past olens[b] are never read.  config: "v1", "v3", a dict or a config.json path
    (`check_config` lists what is refused).  math_mode: "3xf16" (default, fp32-class), "f16", "tf32" or "fp32" for the
    GEMMs.  One host read per call (the device-side length and range checks).  `window` / `stream` /
    `forward(chunk_frames=)` give the same audio in windows of frames (DESIGN.md section 17)."""

    _NAME = "hifigan"

    def __init__(self, config="v1", math_mode: str = "3xf16"):
        super().__init__(math_mode)
        cfg = load_config(config)
        check_config(cfg)
        self.config = cfg
        add_layers(self, cfg)
        self._layers = [m for m in self.modules() if isinstance(m, _WNConv)]      # state_dict order

    def _c_config(self) -> _lib.HiFiGANConfig:
        return c_config(self.config)

    def _load(self, h, device: torch.device) -> None:
        self._load_layers("fs2_hifigan_load", h, device)
