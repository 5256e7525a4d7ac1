"""`FeedForwardTransformer` -- drop-in for the class of the same name in the reference's
fastspeech.py (:28-387), with the mel-synthesis forward path running on libfs2b200.so.

Surface kept from the reference (SURVEY.md section 8b):
  __init__(idim, odim, hp)          hp = the reference's HParam Dotdict (or any mapping)
  forward(xs, ilens, ys, olens, ds, es, ps) -> (loss, report_keys)     fastspeech.py:245-337
  inference(x) -> [L, odim]                                            fastspeech.py:339-357
  _forward(xs, ilens, olens=None, ds=None, es=None, ps=None, is_inference=False) -> 5-tuple
  nn.Module behaviour: parameters()/state_dict()/load_state_dict() with the reference's 225
  keys, .to(), .eval()/.train().

The sub-modules below are *parameter holders* laid out so that `state_dict()` has the
reference's keys in the reference's order; they carry no PyTorch compute graph.  All
arithmetic happens in hand-written sm_90a kernels behind the C ABI (include/fs2_b200.h).
There is no CPU path and no PyTorch fallback: CPU tensors or a missing library raise.
`forward()` in train mode (`model.train()`, train_fastspeech.py:100-123) runs the train path of
fastspeech2_b200/train.py: dropout, BatchNorm batch statistics and a backward through every stage,
all on the library's kernels with torch.autograd as the graph only; `_forward` / `inference` in train
mode raise (the reference's scripts call those under `model.eval()`).

Precision (`precision=` / FS2_PRECISION): "3xf16" (default; alias "3xtf32") is the reference-precision
mode -- every contraction, attention included, error-compensated on the tensor cores, fp32-class
results; "f16" and "tf32" are the 10-bit-mantissa fast modes for the decoder side; "fp32" is exact
fp32 FMA on CUDA cores (include/fs2_b200.h, FS2_MATH_*).  `precision` governs eval only.

Train precision (`train_precision=` / FS2_TRAIN_PRECISION): "fp32" (default) trains in fp32 on CUDA cores; "tf32" runs
every convolution and projection of the train step (forward, input and weight gradient) on the tensor cores in tf32
with fp32 accumulation, as cuDNN does for a reference user's Conv1d by default.  Attention, the norms and the rest of
the step stay fp32 (DESIGN.md §10).

Train attention (`train_attention=` / FS2_TRAIN_ATTENTION): "materialized" (default) runs the train step's attention as
fp32 batched products over a stored [B, heads, L, L] score tensor; "flash" (needs train_precision="tf32") runs it on
fused tf32 tensor-core kernels that store only the row log-sum-exp (DESIGN.md §13).

Deterministic training (`train_deterministic=` / FS2_TRAIN_DETERMINISTIC=1): every gradient, the loss and report, the
BatchNorm running statistics and so the optimizer state are summed in a fixed order, so the same weights, batches and
`torch.manual_seed` give the same bits on every run (DESIGN.md §26).  Off by default: its sums round differently from
the default path's.  A step also runs this way whenever `torch.are_deterministic_algorithms_enabled()`.  It covers the
eval-mode `forward` loss as well.
"""
from __future__ import annotations

import ctypes as C
import inspect
import os
from typing import Any, Dict, List, Optional, Sequence, Tuple

import torch
from torch import nn

from . import _lib
from . import length_regulator as _lr
from .weights import ModelDims, positional_table, variance_bins

DEFAULT_PRECISION = os.environ.get("FS2_PRECISION", "3xf16")
TRAIN_PRECISIONS = ("fp32", "tf32")
TRAIN_ATTENTIONS = ("materialized", "flash")
FLASH_HEAD_WIDTHS = (128, 192)


def resolve_train_precision(train_precision: Optional[str] = None) -> str:
    """The train path's math mode: the argument, else FS2_TRAIN_PRECISION, else "fp32".  "fp32" is fp32 on CUDA cores;
    "tf32" runs every convolution and projection of the train step on the tensor cores (DESIGN.md §10)."""
    mode = train_precision or os.environ.get("FS2_TRAIN_PRECISION") or "fp32"
    if mode in ("f16", "3xf16", "3xtf32"):
        raise ValueError(f"train_precision={mode!r} is not supported: the {mode} kernels read fixed-scale fp16 operand planes, "
                         "which cannot hold gradients without underflow; use 'fp32' or 'tf32'")
    if mode not in TRAIN_PRECISIONS:
        raise ValueError(f"train_precision must be one of {list(TRAIN_PRECISIONS)}, got {mode!r}")
    return mode


def resolve_train_attention(train_attention: Optional[str] = None, train_precision: str = "fp32") -> str:
    """The train step's attention: the argument, else FS2_TRAIN_ATTENTION, else "materialized".  "flash" runs on the fused
    tf32 kernels (DESIGN.md §13), so it needs train_precision="tf32"."""
    mode = train_attention or os.environ.get("FS2_TRAIN_ATTENTION") or "materialized"
    if mode not in TRAIN_ATTENTIONS:
        raise ValueError(f"train_attention must be one of {list(TRAIN_ATTENTIONS)}, got {mode!r}")
    if mode == "flash" and train_precision != "tf32":
        raise ValueError(f"train_attention='flash' needs train_precision='tf32', got {train_precision!r}: the fused attention's products "
                         "are 1xTF32 on the tensor cores, which the fp32 train mode does not allow (it has no fp32-class flash kernel)")
    return mode


def resolve_train_deterministic(train_deterministic: Optional[bool] = None) -> bool:
    """The model's deterministic train mode: the argument, else FS2_TRAIN_DETERMINISTIC ("1" / "true" / "yes" / "on" turn it
    on; "", "0", "false", "no", "off" leave it off).  torch.use_deterministic_algorithms(True) turns a step deterministic
    regardless (train.deterministic_step), so False here never overrides torch's flag."""
    if train_deterministic is not None:
        if not isinstance(train_deterministic, bool):
            raise ValueError(f"train_deterministic must be a bool or None, got {train_deterministic!r}")
        return train_deterministic
    v = os.environ.get("FS2_TRAIN_DETERMINISTIC", "").strip().lower()
    if v in ("1", "true", "yes", "on"):
        return True
    if v in ("", "0", "false", "no", "off"):
        return False
    raise ValueError(f"FS2_TRAIN_DETERMINISTIC must be 1 or 0 (true / false), got {v!r}")


def _get(node: Any, key: str, default: Any = None) -> Any:
    if isinstance(node, dict):
        return node.get(key, default)
    return getattr(node, key, default)


def dims_from_hp(idim: int, odim: int, hp: Any) -> ModelDims:
    """Read the shape-defining subset of `hp` (fastspeech.py:53-160) and reject what the kernels
    do not implement, loudly."""
    m, d = _get(hp, "model"), _get(hp, "data")
    if m is None or d is None:
        raise ValueError("hp must provide .model and .data (utils/hparams.py HParam)")

    def need(cond: bool, what: str):
        if not cond:
            raise NotImplementedError(f"fastspeech2_b200 supports the configs/default.yaml architecture only: {what}")

    need(_get(m, "positionwise_layer_type", "conv1d") == "conv1d", "positionwise_layer_type must be 'conv1d'")
    need(not _get(m, "encoder_normalize_before", False) and not _get(m, "decoder_normalize_before", False), "post-LN blocks only")
    need(not _get(m, "encoder_concat_after", False) and not _get(m, "decoder_concat_after", False), "concat_after=False only")
    need(bool(_get(m, "use_scaled_pos_enc", True)), "use_scaled_pos_enc=True only")
    need(bool(_get(m, "use_batch_norm", True)), "use_batch_norm=True only")
    need(int(_get(m, "reduction_factor", 1)) == 1, "reduction_factor=1 only")
    need(int(_get(m, "postnet_layers", 5)) >= 1, "postnet_layers >= 1")
    # Energy/PitchPredictor ignore hp and are always VariancePredictor(idim) = 2 x 256 x k3
    # (variance_predictor.py:125,198); the kernels share one predictor shape, so the duration predictor must match it
    need((int(_get(m, "duration_predictor_layers")), int(_get(m, "duration_predictor_chans")), int(_get(m, "duration_predictor_kernel_size"))) == (2, 256, 3),
         "duration_predictor_{layers,chans,kernel_size} must be (2, 256, 3), the fixed shape of the energy / pitch predictors")
    return ModelDims(
        idim=int(idim), odim=int(odim), adim=int(_get(m, "adim")),
        aheads=int(_get(m, "aheads")), elayers=int(_get(m, "elayers")), eunits=int(_get(m, "eunits")),
        ddim=int(_get(m, "ddim")), dlayers=int(_get(m, "dlayers")), dunits=int(_get(m, "dunits")),
        ffn_kernel=int(_get(m, "positionwise_conv_kernel_size")),
        # DurationPredictor honours hp; Energy/PitchPredictor hard-code VariancePredictor(idim)
        # defaults 2 x 256 x k3 (variance_predictor.py:125,198).  One shape for all three is
        # what default.yaml yields; anything else was rejected above.
        pred_layers=int(_get(m, "duration_predictor_layers")), pred_chans=int(_get(m, "duration_predictor_chans")),
        pred_kernel=int(_get(m, "duration_predictor_kernel_size")),
        postnet_layers=int(_get(m, "postnet_layers")), postnet_chans=int(_get(m, "postnet_chans")),
        postnet_filts=int(_get(m, "postnet_filts")),
        e_min=float(_get(d, "e_min")), e_max=float(_get(d, "e_max")), p_min=float(_get(d, "p_min")), p_max=float(_get(d, "p_max")),
    )


# ------------------------------------------------------------------------------------------------
# parameter holders (checkpoint layout only)
# ------------------------------------------------------------------------------------------------
class _Holder(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("parameter holder: the forward path runs in libfs2b200.so, not in torch modules")


class _ScaledPosEnc(_Holder):
    def __init__(self, d_model: int, max_len: int):
        super().__init__()
        self.alpha = nn.Parameter(torch.tensor(1.0))
        self.register_buffer("pe", positional_table(max_len, d_model))


class _SelfAttn(_Holder):
    def __init__(self, C_: int):
        super().__init__()
        self.linear_q, self.linear_k = nn.Linear(C_, C_), nn.Linear(C_, C_)
        self.linear_v, self.linear_out = nn.Linear(C_, C_), nn.Linear(C_, C_)


class _ConvFFN(_Holder):
    def __init__(self, C_: int, H: int, k: int):
        super().__init__()
        self.w_1 = nn.Conv1d(C_, H, k, padding=(k - 1) // 2)
        self.w_2 = nn.Conv1d(H, C_, 1)


class _FFTBlock(_Holder):
    def __init__(self, C_: int, H: int, k: int):
        super().__init__()
        self.self_attn = _SelfAttn(C_)
        self.feed_forward = _ConvFFN(C_, H, k)
        self.norm1, self.norm2 = nn.LayerNorm(C_), nn.LayerNorm(C_)
        self.concat_linear = nn.Linear(2 * C_, C_)  # present in the checkpoint, unused (concat_after=False)


class _FFTStack(_Holder):
    def __init__(self, embed: nn.Sequential, C_: int, H: int, k: int, n: int):
        super().__init__()
        self.after_norm = nn.LayerNorm(C_)  # present in the checkpoint, unused (normalize_before=False)
        self.embed = embed
        self.encoders_ = nn.ModuleList([_FFTBlock(C_, H, k) for _ in range(n)])


class _ChannelNorm(_Holder):
    def __init__(self, n: int):
        super().__init__()
        self.layer_norm = nn.LayerNorm(n, eps=1e-12)


class _ConvPredictor(_Holder):
    def __init__(self, cin: int, layers: int, chans: int, k: int):
        super().__init__()
        self.conv = nn.ModuleList([
            nn.Sequential(nn.Conv1d(cin if i == 0 else chans, chans, k, padding=(k - 1) // 2), nn.ReLU(), _ChannelNorm(chans),
                          nn.Dropout(0.5)) for i in range(layers)])
        self.linear = nn.Linear(chans, 1)


class _BinnedPredictor(_Holder):
    """Energy / Pitch predictor: bins buffer + conv predictor (variance_predictor.py:98-232)."""

    def __init__(self, bins_name: str, bins: torch.Tensor, dims: ModelDims):
        super().__init__()
        self.register_buffer(bins_name, bins)
        self.predictor = _ConvPredictor(dims.adim, dims.pred_layers, dims.pred_chans, dims.pred_kernel)
        self._bins_name = bins_name
        self._n_bins = dims.n_bins

    def to_one_hot(self, x: torch.Tensor) -> torch.Tensor:
        """bucketize + one_hot(256).float() (variance_predictor.py:154-159 / :227-232) on the GPU kernels."""
        lib = _lib.load()
        bins = getattr(self, self._bins_name)
        xs = x.contiguous().float()
        ids = torch.empty(xs.shape, dtype=torch.int64, device=xs.device)
        st = _lib.stream_ptr(xs.device)
        _lib.check(lib.fs2_bucketize(_lib.ptr(xs), _lib.ptr(bins), bins.numel(), xs.numel(), _lib.ptr(ids), st), "fs2_bucketize")
        out = torch.empty(tuple(xs.shape) + (self._n_bins,), dtype=torch.float32, device=xs.device)
        _lib.check(lib.fs2_one_hot(_lib.ptr(ids), ids.numel(), self._n_bins, _lib.ptr(out), st), "fs2_one_hot")
        return out


class _Postnet(_Holder):
    def __init__(self, dims: ModelDims):
        super().__init__()
        layers = []
        for i in range(dims.postnet_layers):
            cin = dims.odim if i == 0 else dims.postnet_chans
            cout = dims.odim if i == dims.postnet_layers - 1 else dims.postnet_chans
            mods: List[nn.Module] = [nn.Conv1d(cin, cout, dims.postnet_filts, padding=(dims.postnet_filts - 1) // 2, bias=False),
                                     nn.BatchNorm1d(cout)]
            if i < dims.postnet_layers - 1:
                mods.append(nn.Tanh())
            mods.append(nn.Dropout(0.5))
            layers.append(nn.Sequential(*mods))
        self.postnet = nn.ModuleList(layers)


def _init_like_reference(model: nn.Module, init_type: str) -> None:
    """core/modules.py:51-81 `initialize`."""
    if init_type == "pytorch":
        return
    fns = {"xavier_uniform": nn.init.xavier_uniform_, "xavier_normal": nn.init.xavier_normal_,
           "kaiming_uniform": lambda p: nn.init.kaiming_uniform_(p, nonlinearity="relu"),
           "kaiming_normal": lambda p: nn.init.kaiming_normal_(p, nonlinearity="relu")}
    if init_type not in fns:
        raise ValueError("Unknown initialization: " + init_type)
    for p in model.parameters():
        if p.dim() > 1:
            fns[init_type](p.data)
    for p in model.parameters():
        if p.dim() == 1:
            p.data.zero_()
    for m in model.modules():
        if isinstance(m, (nn.Embedding, nn.LayerNorm)):
            m.reset_parameters()


_CONTROL_NAMES = ("speed", "pitch", "energy")


def _controls_for(B: int, T: int, dev: torch.device, controls: Dict[str, Any], ilens: Any = None) -> Optional[Tuple]:
    """Prosody controls -> (speed, pitch, energy), each None or a contiguous float32 [B, T] tensor on `dev`; None when
    no control is given.  A control is a Python number, a [B] tensor (one factor per utterance) or a [B, T] tensor (one
    factor per phoneme; entries at t >= ilens[b] are ignored).  Factors are rounded to fp32 first and must be finite
    and > 0: values on the host are checked here (per-phoneme ones only when `ilens` is on the host too), the rest in
    the caller's single host read (`_control_violations`)."""
    if all(controls[k] is None for k in _CONTROL_NAMES):
        return None
    out = []
    for name in _CONTROL_NAMES:
        v = controls[name]
        if v is None:
            out.append(None)
            continue
        if not torch.is_tensor(v):
            if isinstance(v, bool) or not isinstance(v, (int, float)):
                raise ValueError(f"{name} must be a number or a tensor, got {type(v).__name__}")
            v = torch.tensor(float(v), dtype=torch.float64)      # rounded to fp32 below (1e39 -> inf, 1e-50 -> 0)
        v = v.detach().to(torch.float32)
        used = None                       # host mask of the factors that matter; None: check on the device
        if v.dim() == 0:
            v = v.expand(B, T)
            used = torch.ones((), dtype=torch.bool)
        elif v.dim() == 1 and v.shape[0] == B:
            v = v[:, None].expand(B, T)
            used = torch.ones((), dtype=torch.bool)
        elif tuple(v.shape) != (B, T):
            raise ValueError(f"{name} must be a number, a [B={B}] or a [B={B}, Tmax={T}] tensor, got {tuple(v.shape)}")
        elif torch.is_tensor(ilens) and not ilens.is_cuda and tuple(ilens.shape) == (B,):
            used = torch.arange(T)[None, :] < ilens[:, None]
        if not v.is_cuda and used is not None:
            bad = ~(torch.isfinite(v) & (v > 0)) & used
            if bool(bad.any()):
                raise ValueError(f"{name}: every factor must be finite and > 0 in fp32 (got {float(v[bad][0])})")
        out.append(v.to(dev).contiguous())
    return tuple(out)


def _control_violations(controls: Tuple, ilens: torch.Tensor, T: int) -> torch.Tensor:
    """Device scalar: how many factors of the valid positions (t < ilens[b]) are non-finite or <= 0."""
    valid = torch.arange(T, device=ilens.device)[None, :] < ilens[:, None]
    bad = [(~(torch.isfinite(c) & (c > 0)) & valid).sum() for c in controls if c is not None]
    return torch.stack(bad).sum()


def n_speakers_from_hp(hp: Any) -> int:
    """hp.model.n_speakers: absent, None or 0 is a single-speaker model."""
    v = _get(_get(hp, "model"), "n_speakers", 0)
    if v is None:
        return 0
    if isinstance(v, bool) or not isinstance(v, int) or v < 0:
        raise ValueError(f"hp.model.n_speakers must be an int >= 0, got {v!r}")
    return int(v)


def _speaker_ids(n_speakers: int, speakers: Any, B: int, dev: torch.device) -> Optional[torch.Tensor]:
    """Speakers of a call -> None (single-speaker model) or a contiguous int64 [B] tensor on `dev`.  Everything that needs
    no device read is checked here; ids on the device are range-checked in the caller's single host read."""
    if n_speakers == 0:
        if speakers is not None:
            raise ValueError("speakers were given but the model has no speaker table (hp.model.n_speakers is 0)")
        return None
    if speakers is None:
        raise ValueError(f"the model has {n_speakers} speakers: pass the speaker ids (speakers=)")
    if not torch.is_tensor(speakers) or speakers.dtype != torch.int64:
        raise ValueError(f"speakers must be an int64 tensor, got {getattr(speakers, 'dtype', type(speakers).__name__)}")
    if speakers.dim() != 1 or speakers.shape[0] != B:
        raise ValueError(f"speakers must be [B={B}], got {tuple(speakers.shape)}")
    if not speakers.is_cuda:
        _check_speaker_range(int(((speakers < 0) | (speakers >= n_speakers)).sum()), n_speakers)
    return speakers.to(dev).contiguous()


def _speaker_violations(spk: torch.Tensor, n_speakers: int) -> torch.Tensor:
    """Device scalar: how many ids lie outside [0, n_speakers)."""
    return ((spk < 0) | (spk >= n_speakers)).sum().view(1)


def _check_speaker_range(bad: int, n_speakers: int) -> None:
    if bad:
        raise ValueError(f"speakers: {bad} id(s) outside [0, n_speakers={n_speakers})")


def _one_speaker(speaker: Any) -> Optional[torch.Tensor]:
    """`inference`'s speaker: None, a Python int or a 0-d int64 tensor -> None or a [1] tensor."""
    if speaker is None:
        return None
    if torch.is_tensor(speaker):
        if speaker.dim() != 0:
            raise ValueError(f"speaker must be an int or a 0-d tensor, got shape {tuple(speaker.shape)}")
        return speaker.reshape(1)
    if isinstance(speaker, bool) or not isinstance(speaker, int):
        raise ValueError(f"speaker must be an int or a 0-d int64 tensor, got {type(speaker).__name__}")
    return torch.tensor([speaker], dtype=torch.int64)


SPEMB_INTEGRATION_TYPES = ("add",)


def spk_embed_dim_from_hp(hp: Any) -> int:
    """hp.model.spk_embed_dim: absent, None or 0 is a model without speaker embeddings; else D in [1, 4096].
    hp.model.spk_embed_integration_type, when set, must be "add" (ESPnet2's default)."""
    m = _get(hp, "model")
    kind = _get(m, "spk_embed_integration_type", None)
    if kind is not None and kind not in SPEMB_INTEGRATION_TYPES:
        raise ValueError(f"hp.model.spk_embed_integration_type must be one of {list(SPEMB_INTEGRATION_TYPES)}, got {kind!r}")
    v = _get(m, "spk_embed_dim", 0)
    return _check_spk_embed_dim(0 if v is None else v, "hp.model.spk_embed_dim")


def _check_spk_embed_dim(v: Any, what: str) -> int:
    if isinstance(v, bool) or not isinstance(v, int) or not (v == 0 or 1 <= v <= _lib.FS2_SPEMB_MAX_DIM):
        raise ValueError(f"{what} must be 0 (none) or an int in [1, {_lib.FS2_SPEMB_MAX_DIM}], got {v!r}")
    return int(v)


def _spemb_tensor(D: int, spembs: Any, B: int, dev: torch.device) -> Optional[torch.Tensor]:
    """Speaker embeddings of a call -> None (model without spk_embed_dim) or a contiguous float32 [B, D] tensor on `dev`,
    detached (embeddings are data).  Non-finite values are found on the device (fs2_spemb_project's status bit)."""
    if D == 0:
        if spembs is not None:
            raise ValueError("speaker embeddings were given but the model has no projection (hp.model.spk_embed_dim is 0)")
        return None
    if spembs is None:
        raise ValueError(f"the model takes {D}-dim speaker embeddings: pass them (spembs= / spemb=)")
    if not torch.is_tensor(spembs) or spembs.dtype != torch.float32:
        raise ValueError(f"spembs must be a float32 tensor, got {getattr(spembs, 'dtype', type(spembs).__name__)}")
    if spembs.dim() != 2 or tuple(spembs.shape) != (B, D):
        raise ValueError(f"spembs must be [B={B}, D={D}], got {tuple(spembs.shape)}")
    if spembs.device != dev:
        raise ValueError(f"spembs must be on {dev} with the model's input, got {spembs.device}")
    return spembs.detach().contiguous()


def _one_spemb(spemb: Any) -> Any:
    """`inference`'s spemb [D] -> [1, D] (anything else is left to _spemb_tensor to refuse)."""
    if torch.is_tensor(spemb) and spemb.dim() == 1:
        return spemb[None]
    if torch.is_tensor(spemb):
        raise ValueError(f"spemb must be a [D] tensor, got shape {tuple(spemb.shape)}")
    return spemb


def _check_spemb_status(word: int) -> None:
    if word & _lib.FS2_SPEMB_NONFINITE:
        raise ValueError("spembs: some speaker embedding(s) hold non-finite values, or values so large (above ~1.8e19) that "
                         "their fp32 sum of squares overflows")


def _without(fn, *names: str) -> inspect.Signature:
    """fn's signature without the parameters `names`."""
    sig = inspect.signature(fn)
    return sig.replace(parameters=[p for p in sig.parameters.values() if p.name not in names])


# ------------------------------------------------------------------------------------------------
class FeedForwardTransformer(nn.Module):
    """Feed-forward Transformer TTS (FastSpeech2) on H100.  See module docstring."""

    @classmethod
    def from_checkpoint(cls, checkpoint, hp=None, precision: Optional[str] = None, device=None, train_precision: Optional[str] = None,
                        train_attention: Optional[str] = None, train_deterministic: Optional[bool] = None):
        """Build the model from a reference checkpoint: a path or the loaded dict `{"model": state_dict, "optim": ..,
        "step": .., "hp_str": .., "githash": ..}` that train_fastspeech.py:235-244 writes (or a bare state_dict, the
        `--old_model` case of inference.py:161-163).  `hp` defaults to the checkpoint's own `hp_str` like
        inference.py:148-152; idim is read off the embedding table instead of the text front-end's symbol list."""
        from .hparams import load_hp_str
        if isinstance(checkpoint, (str, bytes, os.PathLike)):
            checkpoint = torch.load(checkpoint, map_location="cpu", weights_only=True)
        sd = checkpoint["model"] if "model" in checkpoint else checkpoint
        if hp is None:
            if "hp_str" not in checkpoint:
                raise ValueError("checkpoint carries no hp_str: pass hp=")
            hp = load_hp_str(checkpoint["hp_str"])
        idim = int(sd["encoder.embed.0.weight"].shape[0])
        odim = int(_get(_get(hp, "audio"), "num_mels"))
        # the speaker count comes from the table: an hp_str written before multi-speaker models lacks the key
        table = sd.get("speaker_embed.weight")
        n_spk = int(table.shape[0]) if table is not None else 0
        n_hp = n_speakers_from_hp(hp)
        if n_hp and n_hp != n_spk:
            raise ValueError(f"hp.model.n_speakers = {n_hp} but the checkpoint's speaker table has {n_spk} rows")
        # and the speaker-embedding width from the projection (DESIGN.md section 27)
        proj = sd.get("spk_embed_proj.weight")
        d_spe = int(proj.shape[1]) if proj is not None else 0
        d_hp = spk_embed_dim_from_hp(hp)
        if d_hp and d_hp != d_spe:
            raise ValueError(f"hp.model.spk_embed_dim = {d_hp} but the checkpoint's spk_embed_proj.weight takes D = {d_spe}")
        model = cls(idim, odim, hp, precision=precision, train_precision=train_precision, train_attention=train_attention,
                    n_speakers=n_spk, train_deterministic=train_deterministic, spk_embed_dim=d_spe)
        model.load_state_dict(sd, strict="model" in checkpoint)
        model.eval()
        return model.to(device) if device is not None else model

    def __init__(self, idim: int, odim: int, hp: Dict, precision: Optional[str] = None, train_precision: Optional[str] = None,
                 train_attention: Optional[str] = None, n_speakers: Optional[int] = None, train_deterministic: Optional[bool] = None,
                 spk_embed_dim: Optional[int] = None):
        super().__init__()
        dims = dims_from_hp(idim, odim, hp)
        self.dims = dims
        self.idim, self.odim = idim, odim
        m = _get(hp, "model")
        self.use_scaled_pos_enc = bool(_get(m, "use_scaled_pos_enc", True))
        self.use_masking = bool(_get(m, "use_masking", True))
        self.use_weighted_masking = bool(_get(m, "use_weighted_masking", False))
        if not self.use_masking or self.use_weighted_masking:
            raise NotImplementedError("loss kernels implement use_masking=True, use_weighted_masking=False (configs/default.yaml:57-58)")
        self.precision = precision or DEFAULT_PRECISION
        if self.precision not in _lib.MATH_MODES:
            raise ValueError(f"precision must be one of {sorted(_lib.MATH_MODES)}")
        self.train_precision = resolve_train_precision(train_precision)
        self.train_attention = resolve_train_attention(train_attention, self.train_precision)
        self.train_deterministic = resolve_train_deterministic(train_deterministic)
        if self.train_attention == "flash":
            for name, width in (("adim", dims.adim), ("ddim", dims.ddim)):
                if width % dims.aheads or width // dims.aheads not in FLASH_HEAD_WIDTHS:
                    raise ValueError(f"train_attention='flash' supports head widths {list(FLASH_HEAD_WIDTHS)}; {name} = {width} with "
                                     f"aheads = {dims.aheads} gives {width / dims.aheads:g}")

        A, D = dims.adim, dims.ddim
        self.encoder = _FFTStack(nn.Sequential(nn.Embedding(idim, A, padding_idx=0), _ScaledPosEnc(A, dims.pe_len)),
                                 A, dims.eunits, dims.ffn_kernel, dims.elayers)
        self.duration_predictor = _ConvPredictor(A, dims.pred_layers, dims.pred_chans, dims.pred_kernel)
        e_bins, p_bins = variance_bins(dims)
        self.energy_predictor = _BinnedPredictor("energy_bins", e_bins, dims)
        self.energy_embed = nn.Linear(dims.n_bins, A)
        self.pitch_predictor = _BinnedPredictor("pitch_bins", p_bins, dims)
        self.pitch_embed = nn.Linear(dims.n_bins, A)
        self.length_regulator = _lr.LengthRegulator()
        self.decoder = _FFTStack(nn.Sequential(nn.Linear(A, D), nn.LayerNorm(D), nn.Dropout(0.2), nn.ReLU(), _ScaledPosEnc(D, dims.pe_len)),
                                 D, dims.dunits, dims.ffn_kernel, dims.dlayers)
        self.postnet = _Postnet(dims)
        self.feat_out = nn.Linear(D, odim)

        _init_like_reference(self, str(_get(m, "transformer_init", "pytorch")))
        self.encoder.embed[-1].alpha.data = torch.tensor(float(_get(m, "initial_encoder_alpha", 1.0)))
        self.decoder.embed[-1].alpha.data = torch.tensor(float(_get(m, "initial_decoder_alpha", 1.0)))
        # multi-speaker (DESIGN.md section 25): one learned vector per speaker added to the encoder output.  Created last, so
        # the reference's 225 keys keep their order, the new key comes after feat_out, and the other parameters draw the
        # same initial values as in a single-speaker model; nn.Embedding's N(0, 1) init, no padding row
        self.n_speakers = n_speakers_from_hp(hp) if n_speakers is None else int(n_speakers)
        if self.n_speakers < 0:
            raise ValueError(f"n_speakers must be >= 0, got {self.n_speakers}")
        if self.n_speakers:
            self.speaker_embed = nn.Embedding(self.n_speakers, A)
        # external speaker embeddings (DESIGN.md section 27): ESPnet2's spk_embed_proj, created after everything else (the
        # speaker table included), so its two keys come last and every other parameter draws the same initial values;
        # nn.Linear's default init
        d_hp = spk_embed_dim_from_hp(hp)
        self.spk_embed_dim = d_hp if spk_embed_dim is None else _check_spk_embed_dim(spk_embed_dim, "spk_embed_dim")
        if self.spk_embed_dim:
            self.spk_embed_proj = nn.Linear(self.spk_embed_dim, A)

        self.postnet_dropout_rate = float(_get(m, "postnet_dropout_rate", 0.5))
        self.duration_dropout_rate = float(_get(m, "duration_predictor_dropout_rate", 0.1))
        self.dropout_masks = None           # train.MaskSource override (tests inject the reference's masks)
        self._epoch = 0
        self._sd_cache: Optional[list] = None
        self._handle: Optional[C.c_void_p] = None
        self._handle_device: Optional[torch.device] = None
        self._fingerprint: Optional[Tuple] = None
        self._workspace: Optional[torch.Tensor] = None
        self._keepalive: List[Any] = []

    # -- library plumbing --------------------------------------------------------------------
    def __del__(self):
        try:
            if self._handle is not None:
                _lib.load().fs2_destroy(self._handle)
        except Exception:
            pass

    def _device(self) -> torch.device:
        return self.feat_out.weight.device

    def _current_fingerprint(self) -> Tuple:
        """(data_ptr, _version) of every checkpoint tensor plus the explicit epoch.  In-place writes through `.data`
        (`p.data.copy_()`, EMA, the reference's own `initialize()`) do not bump `_version`: call `invalidate()` after
        such an update (`load_state_dict` and `.to()` / `_apply` do it themselves)."""
        if self._sd_cache is None:
            self._sd_cache = list(self.state_dict(keep_vars=True).values())
        return (self._epoch,) + tuple((t.data_ptr(), t._version) for t in self._sd_cache)

    def invalidate(self) -> None:
        """Force a repack of the checkpoint into the kernel layout on the next forward (after weight updates the
        version counters cannot see).  Captured `GraphedForward` objects refuse to replay afterwards."""
        self._epoch += 1
        self._sd_cache = None

    repack = invalidate

    def load_state_dict(self, *a, **k):
        out = super().load_state_dict(*a, **k)
        self.invalidate()
        return out

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        self.invalidate()
        return out

    def _extend_pe(self, stack: "_FFTStack", n: int) -> None:
        """core/embedding.py:48-66 `extend_pe`: regenerate a longer sinusoid table when the input outgrows it."""
        pos = stack.embed[-1]
        if pos.pe.shape[1] >= n:
            return
        pos.pe = positional_table(n, pos.pe.shape[2]).to(device=pos.pe.device, dtype=pos.pe.dtype)
        self.invalidate()

    def _ready(self, like: torch.Tensor) -> C.c_void_p:
        """Handle with weights packed for the current parameters (repacks after load_state_dict,
        .to(), optimizer steps ...)."""
        if self.training:
            raise NotImplementedError(
                "_forward / inference run the eval-mode path; call model.eval() (the reference's scripts do: inference.py:115, "
                "evaluation.py:19, train_fastspeech.py:152).  In train mode use model(xs, ilens, ys, olens, ds, es, ps), which "
                "runs the train path (dropout, BatchNorm batch statistics, backward).")
        dev = self._device()
        if dev.type != "cuda":
            raise _lib.Fs2Error("model parameters are on %s: the H100 path has no CPU fallback, call model.to('cuda')" % dev)
        if like.device != dev:
            raise _lib.Fs2Error(f"input on {like.device} but model on {dev}")
        lib = _lib.load()
        if self._handle is None or self._handle_device != dev:
            if self._handle is not None:
                lib.fs2_destroy(self._handle)
            d = self.dims
            cfg = _lib.Config(d.idim, d.odim, d.adim, d.aheads, d.elayers, d.eunits, d.ddim, d.dlayers, d.dunits, d.ffn_kernel,
                              d.pred_layers, d.pred_chans, d.pred_kernel, d.postnet_layers, d.postnet_chans, d.postnet_filts,
                              d.n_bins, d.pe_len, _lib.MATH_MODES[self.precision])
            h = C.c_void_p()
            _lib.check(lib.fs2_create(C.byref(h), C.byref(cfg), dev.index if dev.index is not None else torch.cuda.current_device()), "fs2_create")
            self._handle, self._handle_device, self._fingerprint = h, dev, None
        fp = self._current_fingerprint()
        if fp != self._fingerprint:
            sd = self.state_dict(keep_vars=True)
            descs = (_lib.WeightDesc * len(sd))()
            keep = []
            for i, (k, t) in enumerate(sd.items()):
                t = t.detach()
                if t.dtype not in (torch.float32, torch.int64):
                    raise _lib.Fs2Error(f"parameter {k} is {t.dtype}: the path is fp32-only like the reference (variance_predictor.py:159)")
                t = t.contiguous()
                keep.append(t)
                name = k.encode()
                keep.append(name)
                shape = (C.c_int64 * 4)(*([int(s) for s in t.shape] + [0] * (4 - t.dim())))
                descs[i] = _lib.WeightDesc(name, t.data_ptr(), t.dim(), shape, 0 if t.dtype == torch.float32 else 1)
            _lib.check(lib.fs2_load_weights(self._handle, descs, len(sd), _lib.stream_ptr(dev)), "fs2_load_weights")
            self._fingerprint = fp
        _lib.check(lib.fs2_set_math_mode(self._handle, _lib.MATH_MODES[self.precision]), "fs2_set_math_mode")
        return self._handle

    def _ws(self, B: int, T: int, L: int) -> torch.Tensor:
        lib = _lib.load()
        need = C.c_size_t()
        _lib.check(lib.fs2_workspace_bytes(self._handle, B, T, L, C.byref(need)), "fs2_workspace_bytes")
        dev = self._device()
        if self._workspace is None or self._workspace.device != dev or self._workspace.numel() < need.value:
            self._workspace = None
            self._workspace = torch.empty(int(need.value), dtype=torch.uint8, device=dev)
        return self._workspace

    # -- the path ----------------------------------------------------------------------------
    def _forward(self, xs: torch.Tensor, ilens: torch.Tensor, olens: torch.Tensor = None, ds: torch.Tensor = None,
                 es: torch.Tensor = None, ps: torch.Tensor = None, is_inference: bool = False,
                 _one_hot: bool = True, _defer_check: Optional[list] = None, _after_out: Optional[torch.Tensor] = None,
                 per_utterance: bool = False, _olens_out: Optional[list] = None,
                 _controls: Optional[Tuple] = None, speakers: Optional[torch.Tensor] = None,
                 spembs: Optional[torch.Tensor] = None) -> Sequence[torch.Tensor]:
        """The reference's `_forward` (fastspeech.py:169-243).  `per_utterance=True` (not in the reference) makes every
        utterance's result independent of its batch mates: utterance b is bit-identical to the B = 1 call on
        `xs[b:b+1, :ilens[b]]` (teacher-forced: with its es / ps sliced to olens[b]), in inference the decoder is masked by
        the predicted lengths, every padded position of every returned tensor is exactly 0 (all-zero one-hot rows), and
        row tiles wholly in padding are skipped.  It needs 1 <= ilens[b] <= Tmax, and in teacher-forced mode
        olens[b] == sum(ds[b, :ilens[b]]).  `_olens_out` (list): receives the olens the decoder ran with.
        `_controls` (from `_controls_for`): prosody factors (speed, pitch, energy) per phoneme, in inference only, and
        only where an utterance's result does not depend on its batch mates (per_utterance, or B = 1); the returned
        durations are then the frame counts actually expanded.  `speakers` (multi-speaker models, DESIGN.md section 25):
        int64 [B] ids in [0, n_speakers); E[speakers[b]] is added to the encoder output at every row (reference semantics)
        or at rows t < ilens[b] (per_utterance).  `spembs` (models with spk_embed_dim = D, DESIGN.md section 27): float32
        [B, D] on the device; W . normalize(spembs[b]) + bias is added after the table, over the same rows."""
        # the handle-less ABI stages (LengthRegulator, losses, ...) run on the CURRENT device like any CUDA library call:
        # select the device the data lives on for the whole call, leave the caller's current device untouched
        if xs.is_cuda and torch.cuda.current_device() != (xs.device.index or 0):
            with torch.cuda.device(xs.device):
                return self._forward(xs, ilens, olens, ds, es, ps, is_inference, _one_hot, _defer_check, _after_out,
                                     per_utterance, _olens_out, _controls, speakers, spembs)
        if _controls is not None:
            if not is_inference:
                raise ValueError("prosody controls apply to inference only (teacher-forced durations, energy and pitch are given)")
            if not per_utterance and xs.shape[0] != 1:
                raise ValueError("prosody controls on a batch need per_utterance=True (use synthesize): under the reference's "
                                 "batch semantics an utterance's result depends on its batch mates")
        if per_utterance:
            self._check_ilens(xs, ilens)
        if xs.dim() != 2:
            raise ValueError("xs must be [B, Tmax]")
        spk = _speaker_ids(self.n_speakers, speakers, int(xs.shape[0]), xs.device)
        spe = _spemb_tensor(self.spk_embed_dim, spembs, int(xs.shape[0]), xs.device)
        h = self._ready(xs)
        lib = _lib.load()
        dev, d = xs.device, self.dims
        st = _lib.stream_ptr(dev)
        flags = _lib.FS2_PER_UTTERANCE if per_utterance else 0
        if xs.dim() != 2:
            raise ValueError("xs must be [B, Tmax]")
        B, T = xs.shape
        if T > self.encoder.embed[-1].pe.shape[1] or (es is not None and es.dim() == 2 and es.shape[1] > self.decoder.embed[-1].pe.shape[1]):
            self._extend_pe(self.encoder, T)
            if es is not None and es.dim() == 2:
                self._extend_pe(self.decoder, int(es.shape[1]))
            h = self._ready(xs)
        xs = xs.to(torch.int64).contiguous()
        ilens = ilens.to(device=dev, dtype=torch.int64).contiguous()
        f32 = dict(dtype=torch.float32, device=dev)

        if is_inference:
            L_known = None
        else:
            if olens is None or ds is None or es is None or ps is None:
                raise ValueError("teacher-forced _forward needs olens, ds, es and ps (fastspeech.py:197-216)")
            L_known = int(es.shape[1])
            if ps.shape != es.shape or es.shape[0] != B:
                raise ValueError(f"es {tuple(es.shape)} / ps {tuple(ps.shape)} must both be [B, Lmax]")

        # stage 1: encoder + duration predictor
        ws = self._ws(B, T, L_known or 0)
        hs = torch.empty((B, T, d.adim), **f32)
        d_log = None if is_inference else torch.empty((B, T), **f32)
        d_int = torch.empty((B, T), dtype=torch.int64, device=dev) if is_inference else None
        if spe is None:
            _lib.check(lib.fs2_encode_spk(h, _lib.ptr(xs), _lib.ptr(ilens), _lib.ptr(spk), B, T, _lib.ptr(hs), _lib.ptr(d_log),
                                          _lib.ptr(d_int), _lib.ptr(ws), ws.numel(), flags, st), "fs2_encode_spk")
        else:
            spe_status = torch.zeros((1,), dtype=torch.int32, device=dev)
            _lib.check(lib.fs2_encode_spemb(h, _lib.ptr(xs), _lib.ptr(ilens), _lib.ptr(spk), _lib.ptr(spe), self.spk_embed_dim, B, T,
                                            _lib.ptr(hs), _lib.ptr(d_log), _lib.ptr(d_int), _lib.ptr(ws), ws.numel(), flags, None,
                                            _lib.ptr(spe_status), st), "fs2_encode_spemb")

        # stage 2: length regulator
        speed, pitch, energy = _controls if _controls is not None else (None, None, None)
        if speed is not None:       # scaled durations on a private copy; d_int then reports the frames actually expanded
            d_used = torch.empty((B, T), dtype=torch.int64, device=dev)
            cum, olens_lr, stats, _ = _lr.plan(hs, d_int, ilens, 1.0, alpha_v=speed, d_used=d_used)
            d_int = d_used
        else:
            cum, olens_lr, stats, _ = _lr.plan(hs, d_int if is_inference else ds, ilens, 1.0)
        if is_inference:
            words = [stats]
            if per_utterance:       # the ilens range rides along in the same transfer
                words.append(torch.stack([ilens.min(), ilens.max()]))
            if _controls is not None:
                words.append(_control_violations(_controls, ilens, T).view(1))
            if spk is not None:     # and the speaker range
                words.append(_speaker_violations(spk, self.n_speakers))
            if spe is not None:     # and the embeddings' status word
                words.append(spe_status.to(torch.int64))
            vals = torch.cat(words).tolist() if len(words) > 1 else stats.tolist()  # the single host sync of inference
            if spe is not None:
                _check_spemb_status(vals.pop())
            if spk is not None:
                _check_speaker_range(vals.pop(), self.n_speakers)
            if _controls is not None and vals[-1]:
                raise ValueError(f"prosody controls: {vals[-1]} factor(s) are non-finite or <= 0 (each must be finite and > 0)")
            if per_utterance:
                self._check_ilens_range(vals[2], vals[3], T)
            L = int(vals[0])
            if L <= 0:
                raise RuntimeError("inference produced zero frames")
            if L > _lr.INT32_MAX:
                raise ValueError(f"an utterance expands to {L} frames, more than the length plan's int32 prefix sum holds")
            if L > self.decoder.embed[-1].pe.shape[1]:
                self._extend_pe(self.decoder, L)
                h = self._ready(xs)
            # reference semantics: decoder unmasked, fastspeech.py:221-224; per-utterance: masked by the planned lengths
            olens_dec = olens_lr if per_utterance else None
        else:
            L = L_known
            olens_dec = olens.to(device=dev, dtype=torch.int64).contiguous()
        if _olens_out is not None:
            _olens_out.append(olens_lr if is_inference else olens_dec)
        fac = None
        if pitch is not None or energy is not None:   # per-phoneme factors -> per-frame, in the gather's pass
            ones = torch.ones((B, T), **f32)
            fac = torch.empty((2, B, L), **f32)
            hm = _lr.gather(hs, cum, ilens, L, torch.stack([energy if energy is not None else ones,
                                                            pitch if pitch is not None else ones]), fac)
        else:
            hm = _lr.gather(hs, cum, ilens, L)

        # stage 3: variance adaptor + decoder + postnet
        ws = self._ws(B, T, L)
        before = torch.empty((B, L, d.odim), **f32)
        if _after_out is not None:      # caller-provided destination of the final mels, e.g. this rank's slot of the root rank's
            after = _after_out          # receive buffer mapped over NVLink (sharded.PeerGather): the last Postnet epilogue stores there
            if tuple(after.shape) != (B, L, d.odim) or after.dtype != torch.float32 or not after.is_contiguous():
                raise ValueError(f"_after_out must be a contiguous float32 [{B}, {L}, {d.odim}] tensor")
        else:
            after = torch.empty((B, L, d.odim), **f32)
        e_out, p_out = torch.empty((B, L), **f32), torch.empty((B, L), **f32)
        want_ids = is_inference and _one_hot
        e_ids = torch.empty((B, L), dtype=torch.int64, device=dev) if want_ids else None
        p_ids = torch.empty((B, L), dtype=torch.int64, device=dev) if want_ids else None
        es_c = None if is_inference else es.to(**f32).contiguous()
        ps_c = None if is_inference else ps.to(**f32).contiguous()
        e_scale = fac[0] if energy is not None else None
        p_scale = fac[1] if pitch is not None else None
        _lib.check(lib.fs2_decode_ctl(h, _lib.ptr(hm), _lib.ptr(olens_dec), _lib.ptr(es_c), _lib.ptr(ps_c), B, L, _lib.ptr(before),
                                      _lib.ptr(after), _lib.ptr(e_out), _lib.ptr(p_out), _lib.ptr(e_ids), _lib.ptr(p_ids),
                                      _lib.ptr(e_scale), _lib.ptr(p_scale), _lib.ptr(ws), ws.numel(), flags, st), "fs2_decode_ctl")

        if is_inference:
            if not _one_hot:
                return before, after, d_int, None, None
            oh_e = torch.empty((B, L, d.n_bins), **f32)
            oh_p = torch.empty((B, L, d.n_bins), **f32)
            _lib.check(lib.fs2_one_hot(_lib.ptr(e_ids), B * L, d.n_bins, _lib.ptr(oh_e), st), "fs2_one_hot")
            _lib.check(lib.fs2_one_hot(_lib.ptr(p_ids), B * L, d.n_bins, _lib.ptr(oh_p), st), "fs2_one_hot")
            return before, after, d_int, oh_e, oh_p

        # teacher-forced: validate what the reference would have tripped over with shape errors
        # (mask widths are max(lengths): utils/util.py:262-272), one host read at the end.
        chk_dev = torch.stack([stats[0], stats[1], ilens.max(), olens_dec.max()])
        if spk is not None:     # the speaker range rides in the same transfer
            chk_dev = torch.cat([chk_dev, _speaker_violations(spk, self.n_speakers)])
        if spe is not None:     # and the embeddings' status word, last
            chk_dev = torch.cat([chk_dev, spe_status.to(torch.int64)])
        if _defer_check is not None:          # CUDA-graph capture: no host read here, the caller validates after replay
            _defer_check.append((chk_dev, T, L))
            return before, after, d_log, e_out, p_out
        if per_utterance:   # + the ilens range and olens == sum(ds) (the zero rows of hm end at sum(ds)), same transfer
            chk = torch.cat([chk_dev, torch.stack([ilens.min(), (olens_dec != olens_lr).sum()])]).tolist()
            self._check_ilens_range(chk[-2], chk[2], T)
            if chk[-1]:
                raise ValueError(f"per_utterance: olens differs from sum(ds) in {chk[-1]} utterance(s)")
        else:
            chk = chk_dev.tolist()
        if spe is not None:
            _check_spemb_status(chk[4 + (spk is not None)])
        if spk is not None:
            _check_speaker_range(chk[4], self.n_speakers)
        self._validate_lengths(chk[:4], T, L)
        return before, after, d_log, e_out, p_out

    @staticmethod
    def _check_ilens_range(imin: int, imax: int, T: int) -> None:
        if imin < 1 or imax > T:
            raise ValueError(f"per_utterance: every ilens[b] must lie in [1, Tmax={T}] (got min {imin}, max {imax})")

    @classmethod
    def _check_ilens(cls, xs: torch.Tensor, ilens: torch.Tensor) -> None:
        """Argument checks of the per-utterance mode that need no device: shapes, and the ilens range when ilens is on
        the host (lengths on the device are checked in the call's single host read)."""
        if xs.dim() != 2:
            raise ValueError("xs must be [B, Tmax]")
        if not torch.is_tensor(ilens) or ilens.dim() != 1 or ilens.shape[0] != xs.shape[0] or xs.shape[0] == 0:
            raise ValueError(f"ilens must be a non-empty [B] tensor matching xs {tuple(xs.shape)}")
        if not ilens.is_cuda:
            cls._check_ilens_range(int(ilens.min()), int(ilens.max()), int(xs.shape[1]))

    @staticmethod
    def _validate_lengths(chk, T: int, L: int) -> None:
        if chk[1]:
            raise RuntimeError(f"LengthRegulator: {chk[1]} negative duration(s)")
        if chk[2] != T:
            raise RuntimeError(f"xs has Tmax={T} but max(ilens)={chk[2]} (the reference's masks are max(ilens) wide)")
        if chk[0] != L or chk[3] != L:
            raise RuntimeError(f"length mismatch: es/ps have Lmax={L}, max(sum(ds))={chk[0]}, max(olens)={chk[3]}")

    def graphed_forward(self, xs, ilens, olens, ds, es, ps, after_out: Optional[torch.Tensor] = None) -> "GraphedForward":
        """Capture the teacher-forced `_forward` for these shapes into one CUDA graph (see GraphedForward).  `after_out`:
        where the final mels are written (default: a fresh tensor), e.g. a peer-mapped slot of `sharded.PeerGather`."""
        return GraphedForward(self, xs, ilens, olens, ds, es, ps, after_out=after_out)

    def graphed_synthesize(self, B: int, T: int, capacity: int, vocoder=None) -> "GraphedSynthesis":
        """Capture `synthesize` (and `vocoder`, a MelGAN / HiFi-GAN / BigVGAN / iSTFTNet vocoder, when given) for B slots
        of T phonemes at `capacity` frames into one CUDA graph that reads nothing back (see GraphedSynthesis)."""
        return GraphedSynthesis(self, B, T, capacity, vocoder)

    def forward(self, xs: torch.Tensor, ilens: torch.Tensor, ys: torch.Tensor, olens: torch.Tensor, ds: torch.Tensor,
                es: torch.Tensor, ps: torch.Tensor, speakers: Optional[torch.Tensor] = None,
                spembs: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, List[Dict[str, float]]]:
        """Loss computation (fastspeech.py:245-337). Returns (loss, report_keys).  In train mode the loss is attached to
        the autograd graph of the train path (fastspeech2_b200/train.py) so `loss.backward()` fills `.grad` of every
        parameter the reference trains; `self.dropout_masks` (a train.MaskSource) may be set to inject masks.
        `speakers`: int64 [B] ids of a multi-speaker model (required there, refused otherwise).  `spembs`: float32 [B, D]
        speaker embeddings of a model with spk_embed_dim = D (required there, refused otherwise); they get no gradient."""
        if xs.is_cuda and torch.cuda.current_device() != (xs.device.index or 0):
            with torch.cuda.device(xs.device):
                return self.forward(xs, ilens, ys, olens, ds, es, ps, speakers, spembs)
        from .train import deterministic_step, masked_losses, train_forward
        if self.training:
            return train_forward(self, xs, ilens, ys, olens, ds, es, ps, masks=self.dropout_masks, speakers=speakers, spembs=spembs)
        self._ready(xs)
        lib = _lib.load()
        dev = xs.device
        ilens = ilens.to(device=dev, dtype=torch.int64)
        olens = olens.to(device=dev, dtype=torch.int64)
        tmax, lmax = torch.stack([ilens.max(), olens.max()]).tolist()
        xs = xs[:, :tmax]  # fastspeech.py:266-267
        ds_t = ds[:, :tmax].contiguous() if ds.shape[1] != tmax else ds
        es_t, ps_t = es[:, :lmax], ps[:, :lmax]
        before, after, d_outs, e_outs, p_outs = self._forward(xs, ilens, olens, ds_t, es_t, ps_t, is_inference=False,
                                                              speakers=speakers, spembs=spembs)
        if ds_t is not ds and ds_t.shape == ds[:, :tmax].shape:
            ds[:, :tmax].copy_(ds_t)
        B, T = xs.shape
        L = before.shape[1]
        ys_c = ys.to(dtype=torch.float32, device=dev).contiguous()
        es_c, ps_c = es_t.to(torch.float32).contiguous(), ps_t.to(torch.float32).contiguous()
        ds_c = ds_t.contiguous()
        if deterministic_step(self):
            out7 = masked_losses(before, after, d_outs, e_outs, p_outs, ys_c, ds_c, es_c, ps_c, ilens.contiguous(), olens.contiguous(), True)
        else:
            out7 = torch.empty((7,), dtype=torch.float32, device=dev)
            scratch = torch.empty((16,), dtype=torch.float64, device=dev)
            _lib.check(lib.fs2_masked_losses(_lib.ptr(before), _lib.ptr(after), _lib.ptr(ys_c), int(ys_c.shape[1]), _lib.ptr(d_outs),
                                             _lib.ptr(ds_c), _lib.dur_dtype(ds_c), _lib.ptr(e_outs), _lib.ptr(p_outs), _lib.ptr(es_c),
                                             _lib.ptr(ps_c), _lib.ptr(ilens.contiguous()), _lib.ptr(olens.contiguous()), B, T, L,
                                             self.odim, _lib.ptr(out7), _lib.ptr(scratch), _lib.stream_ptr(dev)), "fs2_masked_losses")
        vals = out7.tolist()
        names = ["l1_loss", "before_loss", "after_loss", "duration_loss", "energy_loss", "pitch_loss", "loss"]
        return out7[6], [{k: v} for k, v in zip(names, vals)]

    def inference(self, x: torch.Tensor, speaker=None, spemb=None) -> torch.Tensor:
        """x [T] int64 -> mel [L, odim] (fastspeech.py:339-357).  speaker: the id (an int or a 0-d int64 tensor) of a
        multi-speaker model; spemb: the float32 [D] speaker embedding of a model with spk_embed_dim = D."""
        ilens = torch.tensor([x.shape[0]], dtype=torch.long, device=x.device)
        _, outs, _, _, _ = self._forward(x.unsqueeze(0), ilens, is_inference=True, _one_hot=False, speakers=_one_speaker(speaker),
                                         spembs=_one_spemb(spemb))
        return outs[0]

    # `forward` and `inference` report the reference's signatures to introspection (fastspeech.py:245-254, :339, what
    # drop-in launchers check); `speakers` / `speaker` and `spembs` / `spemb` are extra keywords that only multi-speaker
    # models and models with speaker embeddings use
    forward.__signature__ = _without(forward, "speakers", "spembs")
    inference.__signature__ = _without(inference, "speaker", "spemb")

    def inference_controlled(self, x: torch.Tensor, *, speed=None, pitch=None, energy=None, speaker=None, spemb=None) -> torch.Tensor:
        """`inference` with prosody controls (not in the reference, whose `_forward` passes alpha = 1 to its
        LengthRegulator and pitch / energy predictors; `inference` itself keeps the reference's signature).  Each control
        is None, a number or a [T] tensor of per-phoneme factors, finite and > 0.  speed multiplies the predicted
        durations (> 1 is slower): rint_half_even(fp32(d) * fp32(a)), then the all-zero rule on the scaled slice.  pitch
        and energy multiply the predicted values before bucketize, one fp32 rounding, each frame by the factor of the
        phoneme it was expanded from (pitch is in Hz: 2 ** (k / 12) shifts by k semitones).  With no control this is
        `inference`."""
        if x.dim() != 1:
            raise ValueError("x must be [T]")
        ctl = {"speed": speed, "pitch": pitch, "energy": energy}
        for k, v in ctl.items():
            if torch.is_tensor(v) and v.dim() != 0:
                if v.dim() != 1 or v.shape[0] != x.shape[0]:
                    raise ValueError(f"{k} must be a number or a [T={x.shape[0]}] tensor, got {tuple(v.shape)}")
                ctl[k] = v[None, :]
        controls = _controls_for(1, int(x.shape[0]), x.device, ctl)
        ilens = torch.tensor([x.shape[0]], dtype=torch.long, device=x.device)
        _, outs, _, _, _ = self._forward(x.unsqueeze(0), ilens, is_inference=True, _one_hot=False, _controls=controls,
                                         speakers=_one_speaker(speaker), spembs=_one_spemb(spemb))
        return outs[0]

    def synthesize(self, xs: torch.Tensor, ilens: torch.Tensor, *, speakers=None, speed=None, pitch=None,
                   energy=None, spembs=None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Per-utterance batched inference (not in the reference): xs [B, Tmax] int64 (0 = pad), ilens [B] with
        1 <= ilens[b] <= Tmax -> (mels [B, Lmax, odim], olens [B] int64, durations [B, Tmax] int64), all on the device.
        durations[b], olens[b] and mels[b, :olens[b]] are bit-identical to what `inference(xs[b, :ilens[b]])` computes,
        whatever else is in the batch; mels[b, olens[b]:] and durations[b, ilens[b]:] are 0.  One host read per call.
        speed / pitch / energy: prosody controls as in `inference_controlled`, each None, a number, a [B] tensor (per
        utterance) or a [B, Tmax] tensor (per phoneme; entries past ilens[b] are ignored).  Utterance b is then
        bit-identical to `inference_controlled` on it with its slice of the controls.  durations are the frame counts expanded (after speed and
        the all-zero rule): durations.sum(1) == olens.  speakers: int64 [B] ids of a multi-speaker model; utterance b is
        then bit-identical to `inference` on it with speaker speakers[b].  spembs: float32 [B, D] speaker embeddings of a
        model with spk_embed_dim = D; utterance b is then bit-identical to `inference` on it with spemb=spembs[b]."""
        if xs.dim() != 2:
            raise ValueError("xs must be [B, Tmax]")
        controls = _controls_for(int(xs.shape[0]), int(xs.shape[1]), xs.device,
                                 {"speed": speed, "pitch": pitch, "energy": energy}, ilens)
        got: list = []
        _, after, dur, _, _ = self._forward(xs, ilens, is_inference=True, _one_hot=False, per_utterance=True, _olens_out=got,
                                            _controls=controls, speakers=speakers, spembs=spembs)
        return after, got[0], dur


class GraphedForward:
    """Teacher-forced `_forward` of one fixed shape replayed as a single CUDA graph.

    The ~90 kernel launches of a step (each with its TMA descriptors baked into the launch parameters) are captured
    once; a call copies the inputs into the graph's static buffers (`self.inputs`; callers may also fill those directly
    and call `replay()`), replays, and returns the static output tensors `(before, after, d_outs, e_outs, p_outs)`
    (valid until the next replay).

    Validation of the length words (what the eager path reads back after every forward):
      validate=True        read them now (one host sync per call) and raise like the eager path;
      validate="deferred"  copy them to pinned host memory asynchronously; the check of replay i runs at the start of
                           call i+1 (or in `flush()`), so replays queue back to back with no host bubble;
      validate=False       no check.
    The graph owns references to the workspace and static buffers it was captured with, so later eager calls that grow
    the model's workspace cannot hand that memory to anyone else.  Weight updates require a new capture (the packed
    weight arena is part of the graph): `__call__` raises if the model was repacked or its parameters changed."""

    def __init__(self, model: FeedForwardTransformer, xs, ilens, olens, ds, es, ps, after_out: Optional[torch.Tensor] = None):
        self.model = model
        self._after_out = after_out
        dev = xs.device
        self.inputs = [t.detach().clone().contiguous() for t in (xs, ilens.to(dev), olens.to(dev), ds, es, ps)]
        with torch.no_grad():
            for _ in range(2):                      # warm-up: packs weights, sizes the workspace, sets kernel attributes
                model._forward(*self.inputs, is_inference=False, _after_out=after_out)
            torch.cuda.synchronize(dev)
            self._fingerprint = model._current_fingerprint()
            self._params = list(model._sd_cache)
            self._versions = sum(t._version for t in self._params)
            self._workspace = model._workspace      # keep the captured scratch alive for the life of the graph
            self.graph = torch.cuda.CUDAGraph()
            deferred: list = []
            with torch.cuda.graph(self.graph):
                self.outputs = model._forward(*self.inputs, is_inference=False, _defer_check=deferred, _after_out=after_out)
            self._chk, self._T, self._L = deferred[0]
        self._chk_host = torch.empty(self._chk.shape, dtype=self._chk.dtype).pin_memory()
        self._chk_event = torch.cuda.Event()
        self._pending = False

    def _check_model(self) -> None:
        m = self.model
        if m._epoch != self._fingerprint[0] or sum(t._version for t in self._params) != self._versions:
            raise RuntimeError("model parameters changed since capture: build a new GraphedForward")

    def flush(self) -> None:
        """Run the outstanding deferred validation (waits for the replay it belongs to)."""
        if self._pending:
            self._pending = False
            self._chk_event.synchronize()
            FeedForwardTransformer._validate_lengths(self._chk_host.tolist(), self._T, self._L)

    def replay(self, validate=True):
        """Replay on the current contents of `self.inputs`."""
        self._check_model()
        self.flush()
        self.graph.replay()
        if validate == "deferred":
            self._chk_host.copy_(self._chk, non_blocking=True)
            self._chk_event.record()
            self._pending = True
        elif validate:
            FeedForwardTransformer._validate_lengths(self._chk.tolist(), self._T, self._L)
        return self.outputs

    def __call__(self, xs, ilens, olens, ds, es, ps, validate=True):
        for dst, src in zip(self.inputs, (xs, ilens, olens, ds, es, ps)):
            if dst.shape != src.shape:
                raise ValueError(f"captured for shape {tuple(dst.shape)}, got {tuple(src.shape)}")
            if dst.data_ptr() != src.data_ptr():
                dst.copy_(src, non_blocking=True)
        return self.replay(validate)


class GraphedSynthesis:
    """Per-utterance synthesis (`synthesize`, optionally followed by a neural vocoder) replayed as one CUDA graph at a
    fixed frame capacity, with no host read (DESIGN.md section 21).

    `synthesize` sizes the decoder by Lmax, which it reads back from the device; here every decoder-side buffer is
    `capacity` frames long and the capacity length plan (fs2_length_plan_cap) decides on the device which slots run:
    slot b runs when 1 <= ilens[b] <= T, its control factors are finite and > 0, and need[b] (its planned frame count)
    <= capacity; every other slot is written as exact zeros (its own row tiles are dead, DESIGN.md section 21).  Captured once for B slots of T phonemes,
    the current weights, precision and vocoder:

      encoder + duration predictor -> capacity plan -> gather -> variance adaptor, decoder, Postnet at L = capacity
      [-> vocoder._call at Lmax = capacity] -> status fold

    Static inputs (`self.xs` [B, T], `self.ilens` [B], `self.speed` / `self.pitch` / `self.energy` [B, T] float32, 1.0
    when not set, which is bit-identical to no control; `self.speakers` [B] int64 on a multi-speaker model, whose ids the
    plan checks on the device, so changing only the speakers between replays needs no recapture; `self.spembs` [B, D]
    float32 on a model with speaker embeddings, likewise, whose non-finite slots the plan empties); static outputs, valid until the next replay: mels [B, capacity,
    80], olens [B], durations [B, T] and need [B], and with a vocoder audio [B, capacity * 256] and alens [B] = olens * 256.
    A slot that ran is bit-identical to `synthesize` on that utterance alone (and its audio to the vocoder on that);
    rows past olens[b] and every row of a slot that did not run are +0.

    Validation, as in `GraphedForward`: each replay copies one status word to pinned host memory asynchronously;
    validate=True checks it at once, "deferred" at the next call or `flush()`, False never.  Bad ilens and bad control
    factors raise ValueError as `synthesize` does; the vocoder's range bit raises as the vocoder would.  Overflow is not
    an error: `overflowed()` lists those slots and `need` says what capacity would fit them.  The graph keeps its own
    workspaces; a change of the model's or the vocoder's parameters after capture (or an eager call that grows the
    positional tables, which repacks the weights) makes `__call__` raise."""

    def __init__(self, model: FeedForwardTransformer, B: int, T: int, capacity: int, vocoder=None):
        for name, v in (("B", B), ("T", T), ("capacity", capacity)):
            if isinstance(v, bool) or not isinstance(v, int) or v < 1:
                raise ValueError(f"{name} must be an int >= 1 (got {v!r})")
        if capacity > _lr.INT32_MAX:
            raise ValueError(f"capacity={capacity} exceeds the length plan's int32 prefix sum ({_lr.INT32_MAX})")
        if vocoder is not None:
            from ._kernel_module import NeuralVocoder
            if not isinstance(vocoder, NeuralVocoder) or not hasattr(vocoder, "_chain"):
                raise ValueError(f"vocoder must be a NeuralVocoder upsampling chain (MelGAN, HiFi-GAN, BigVGAN or iSTFTNet), got "
                                 f"{type(vocoder).__name__}: WaveGlow's noise and Griffin-Lim are not captured")
            vocoder._check_size(B, capacity)
        dev = model._device()
        if dev.type != "cuda":
            raise _lib.Fs2Error(f"model parameters are on {dev}: the H100 path has no CPU fallback, call model.to('cuda')")
        self.model, self.vocoder, self.device = model, vocoder, dev
        self.B, self.T, self.capacity = B, T, capacity
        d = model.dims
        i64, f32 = dict(dtype=torch.int64, device=dev), dict(dtype=torch.float32, device=dev)
        self.xs, self.ilens = torch.zeros((B, T), **i64), torch.zeros((B,), **i64)
        self.speakers = torch.zeros((B,), **i64) if model.n_speakers else None
        D = model.spk_embed_dim
        self.spembs = torch.zeros((B, D), **f32) if D else None
        self._spemb_bad = torch.zeros((B,), dtype=torch.int32, device=dev) if D else None
        self.speed = torch.ones((B, T), **f32)
        self._fac = torch.ones((2, B, T), **f32)            # the gather's per-phoneme planes: energy, pitch
        self.energy, self.pitch = self._fac[0], self._fac[1]
        self._controlled = False
        self._hs = torch.empty((B, T, d.adim), **f32)
        self._d_int = torch.empty((B, T), **i64)
        self._cum = torch.empty((B, T), dtype=torch.int32, device=dev)
        self.olens, self.need, self.durations = torch.empty((B,), **i64), torch.empty((B,), **i64), torch.empty((B, T), **i64)
        self._hm = torch.empty((B, capacity, d.adim), **f32)
        self._fac_out = torch.empty((2, B, capacity), **f32)
        self._before, self.mels = torch.empty((B, capacity, d.odim), **f32), torch.empty((B, capacity, d.odim), **f32)
        self._e_out, self._p_out = torch.empty((B, capacity), **f32), torch.empty((B, capacity), **f32)
        self._plan_status = torch.empty((1,), dtype=torch.int32, device=dev)
        self.status = torch.empty((1,), dtype=torch.int32, device=dev)
        self.audio = self.alens = self._voc_status = None
        with torch.no_grad():
            if T > model.encoder.embed[-1].pe.shape[1]:
                model._extend_pe(model.encoder, T)
            if capacity > model.decoder.embed[-1].pe.shape[1]:
                model._extend_pe(model.decoder, capacity)
            self._h = model._ready(self.xs)
            n = C.c_size_t()
            _lib.check(_lib.load().fs2_workspace_bytes(self._h, B, T, capacity, C.byref(n)), "fs2_workspace_bytes")
            self._ws = torch.empty(int(n.value), dtype=torch.uint8, device=dev)
            if vocoder is not None:
                from ._kernel_module import query_bytes
                self._vh = vocoder._handle(dev)
                self._vws = torch.empty(query_bytes(f"fs2_{vocoder._NAME}_workspace_bytes", self._vh, B, capacity),
                                        dtype=torch.uint8, device=dev)
                self.audio = torch.empty((B, capacity * vocoder.HOP), **f32)
                self.alens = torch.empty((B,), **i64)
                self._voc_status = torch.empty((1,), dtype=torch.int32, device=dev)
                self._voc_fingerprint = vocoder._fingerprint()
            with torch.cuda.device(dev):
                for _ in range(2):                  # warm-up on empty slots: kernel attributes, lazily built launch state
                    self._run()
                torch.cuda.synchronize(dev)
                self._fingerprint = model._current_fingerprint()
                self._params = list(model._sd_cache)
                self._versions = sum(t._version for t in self._params)
                self.graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph):
                    self._run()
        self._status_host = torch.empty((1,), dtype=torch.int32).pin_memory()
        self._status_event = torch.cuda.Event()
        self._pending = False

    def _run(self) -> None:
        """The captured sequence, on the static buffers."""
        lib, P = _lib.load(), _lib.ptr
        B, T, Lc, d = self.B, self.T, self.capacity, self.model.dims
        st = _lib.stream_ptr(self.device)
        flags = _lib.FS2_PER_UTTERANCE
        if self.spembs is None:
            _lib.check(lib.fs2_encode_spk(self._h, P(self.xs), P(self.ilens), P(self.speakers), B, T, P(self._hs), None,
                                          P(self._d_int), P(self._ws), self._ws.numel(), flags, st), "fs2_encode_spk")
            _lib.check(lib.fs2_length_plan_cap_spk(P(self._d_int), _lib.FS2_DUR_I64, P(self.ilens), P(self.speed), P(self._fac),
                                                   P(self.speakers), self.model.n_speakers, B, T, Lc, P(self._cum), P(self.olens),
                                                   P(self.need), P(self.durations), P(self._plan_status), st), "fs2_length_plan_cap_spk")
        else:   # a slot whose embedding is non-finite is emptied by the plan, which sets FS2_SPEMB_NONFINITE
            _lib.check(lib.fs2_encode_spemb(self._h, P(self.xs), P(self.ilens), P(self.speakers), P(self.spembs),
                                            self.model.spk_embed_dim, B, T, P(self._hs), None, P(self._d_int), P(self._ws),
                                            self._ws.numel(), flags, P(self._spemb_bad), None, st), "fs2_encode_spemb")
            _lib.check(lib.fs2_length_plan_cap_spemb(P(self._d_int), _lib.FS2_DUR_I64, P(self.ilens), P(self.speed), P(self._fac),
                                                     P(self.speakers), self.model.n_speakers, P(self._spemb_bad), B, T, Lc,
                                                     P(self._cum), P(self.olens), P(self.need), P(self.durations),
                                                     P(self._plan_status), st), "fs2_length_plan_cap_spemb")
        _lib.check(lib.fs2_length_gather_ex(P(self._hs), P(self._cum), P(self.ilens), B, T, d.adim, P(self._hm), Lc, P(self._fac),
                                            P(self._fac_out), st), "fs2_length_gather_ex")
        _lib.check(lib.fs2_decode_ctl(self._h, P(self._hm), P(self.olens), None, None, B, Lc, P(self._before), P(self.mels),
                                      P(self._e_out), P(self._p_out), None, None, P(self._fac_out[0]), P(self._fac_out[1]),
                                      P(self._ws), self._ws.numel(), flags, st), "fs2_decode_ctl")
        hop = 1
        if self.vocoder is not None:
            self.vocoder._call(self._vh, self.mels, self.olens, B, Lc, self.audio, self._voc_status, self._vws)
            hop = self.vocoder.HOP
        _lib.check(lib.fs2_synth_status(P(self._plan_status), P(self._voc_status), P(self.olens), B, hop, P(self.status),
                                        P(self.alens), st), "fs2_synth_status")

    @property
    def outputs(self) -> tuple:
        """(mels, olens, durations), and with a vocoder (..., audio, alens): the static outputs of the last replay."""
        out = (self.mels, self.olens, self.durations)
        return out if self.vocoder is None else out + (self.audio, self.alens)

    @staticmethod
    def check_request(xs, ilens, B: int, T: int) -> Tuple[int, int]:
        """The checks of a request that need no device: xs [b, t] with b <= B, t <= T, and ilens [b] (values in [0, t]
        when on the host; on the device they are checked against T in the status word).  -> (b, t)."""
        if not torch.is_tensor(xs) or xs.dim() != 2 or xs.shape[0] == 0 or xs.shape[1] == 0:
            raise ValueError("xs must be a non-empty [b, t] tensor")
        b, t = int(xs.shape[0]), int(xs.shape[1])
        if b > B or t > T:
            raise ValueError(f"a request of b={b} utterances of t={t} phonemes does not fit the graph's B={B}, T={T}")
        if not torch.is_tensor(ilens) or ilens.dim() != 1 or ilens.shape[0] != b:
            raise ValueError(f"ilens must be a [b={b}] tensor")
        if ilens.dtype.is_floating_point or ilens.dtype == torch.bool:
            raise ValueError("ilens must be an integer tensor")
        if not ilens.is_cuda and b and (int(ilens.min()) < 0 or int(ilens.max()) > t):
            raise ValueError(f"every ilens[b] must lie in [0, t={t}] (0 marks an empty slot)")
        return b, t

    def _check_model(self) -> None:
        m = self.model
        if m._epoch != self._fingerprint[0] or sum(t._version for t in self._params) != self._versions:
            raise RuntimeError("model parameters changed since capture: build a new GraphedSynthesis")
        if self.vocoder is not None and self.vocoder._fingerprint() != self._voc_fingerprint:
            raise RuntimeError("vocoder parameters changed since capture: build a new GraphedSynthesis")

    def _raise_for(self, word: int) -> None:
        if word & _lib.FS2_PLAN_BAD_ILENS:
            raise ValueError(f"every ilens[b] must lie in [0, T={self.T}] (0 marks an empty slot)")
        if word & _lib.FS2_PLAN_BAD_CONTROL:
            raise ValueError("prosody controls: some factor(s) are non-finite or <= 0 (each must be finite and > 0)")
        if word & _lib.FS2_PLAN_BAD_SPEAKER:
            _check_speaker_range(1, self.model.n_speakers)
        _check_spemb_status(word)
        voc = word >> _lib.FS2_SYNTH_VOC_SHIFT
        if voc and self.vocoder is not None:
            for bit, message in self.vocoder._status_table():
                if voc & bit:
                    raise ValueError(message)

    def flush(self) -> None:
        """Run the outstanding deferred validation (waits for the replay it belongs to)."""
        if self._pending:
            self._pending = False
            self._status_event.synchronize()
            self._raise_for(int(self._status_host[0]))

    def replay(self, validate=True) -> tuple:
        """Replay on the current contents of the static inputs; -> `outputs`."""
        self._check_model()
        self.flush()
        with torch.cuda.device(self.device):
            self.graph.replay()
            if validate:
                self._status_host.copy_(self.status, non_blocking=True)
                self._status_event.record()
                self._pending = True
        if validate and validate != "deferred":
            self.flush()
        return self.outputs

    def __call__(self, xs, ilens, speakers=None, speed=None, pitch=None, energy=None, validate=True, spembs=None) -> tuple:
        """Synthesize b <= B requests of t <= T phonemes: xs [b, t] (0 = pad) and ilens [b] are copied into slots 0 .. b-1,
        slots b .. B-1 become empty.  speakers: int64 [b] ids of a multi-speaker model (ids on the device are checked in the
        status word).  speed / pitch / energy: None, a number, a [b] or a [b, t] tensor, as in `synthesize`.  spembs:
        float32 [b, D] speaker embeddings of a model with spk_embed_dim = D, copied into the static `self.spembs`; a
        non-empty slot with a non-finite embedding comes out as zeros and the status word raises ValueError.
        -> `outputs` (all B slots)."""
        if validate not in (True, False, "deferred"):
            raise ValueError(f"validate must be True, False or 'deferred' (got {validate!r})")
        self._check_model()
        b, t = self.check_request(xs, ilens, self.B, self.T)
        spk = _speaker_ids(self.model.n_speakers, speakers, b, self.device)
        spe = _spemb_tensor(self.model.spk_embed_dim, spembs, b, self.device)
        controls = _controls_for(b, t, self.device, {"speed": speed, "pitch": pitch, "energy": energy}, ilens)
        with torch.cuda.device(self.device):
            self.xs.zero_()
            self.xs[:b, :t].copy_(xs, non_blocking=True)
            self.ilens.zero_()
            self.ilens[:b].copy_(ilens, non_blocking=True)
            if spk is not None:
                self.speakers.zero_()
                self.speakers[:b].copy_(spk, non_blocking=True)
            if spe is not None:
                self.spembs.zero_()
                self.spembs[:b].copy_(spe, non_blocking=True)
            if self._controlled or controls is not None:     # factors stay 1.0 between uncontrolled requests
                self.speed.fill_(1.0)
                self._fac.fill_(1.0)
                for dst, src in zip((self.speed, self.pitch, self.energy), controls or (None,) * 3):
                    if src is not None:
                        dst[:b, :t].copy_(src)
                self._controlled = controls is not None
        return self.replay(validate)

    def overflowed(self) -> List[int]:
        """The slots of the last replay whose planned frames (need) exceed the capacity: they were skipped (olens 0), not
        refused.  One host read."""
        need, il = torch.stack([self.need, self.ilens]).tolist()
        return [b for b in range(self.B) if 1 <= il[b] <= self.T and need[b] > self.capacity]
