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
"""
from __future__ import annotations

import ctypes as C
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


# ------------------------------------------------------------------------------------------------
class FeedForwardTransformer(nn.Module):
    """Feed-forward Transformer TTS (FastSpeech2) on H100.  See module docstring."""

    @classmethod
    def from_checkpoint(cls, checkpoint, hp=None, precision: Optional[str] = None, device=None, train_precision: Optional[str] = None,
                        train_attention: Optional[str] = None):
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
        model = cls(idim, odim, hp, precision=precision, train_precision=train_precision, train_attention=train_attention)
        model.load_state_dict(sd, strict="model" in checkpoint)
        model.eval()
        return model.to(device) if device is not None else model

    def __init__(self, idim: int, odim: int, hp: Dict, precision: Optional[str] = None, train_precision: Optional[str] = None,
                 train_attention: Optional[str] = None):
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
                 _controls: Optional[Tuple] = None) -> Sequence[torch.Tensor]:
        """The reference's `_forward` (fastspeech.py:169-243).  `per_utterance=True` (not in the reference) makes every
        utterance's result independent of its batch mates: utterance b is bit-identical to the B = 1 call on
        `xs[b:b+1, :ilens[b]]` (teacher-forced: with its es / ps sliced to olens[b]), in inference the decoder is masked by
        the predicted lengths, every padded position of every returned tensor is exactly 0 (all-zero one-hot rows), and
        row tiles wholly in padding are skipped.  It needs 1 <= ilens[b] <= Tmax, and in teacher-forced mode
        olens[b] == sum(ds[b, :ilens[b]]).  `_olens_out` (list): receives the olens the decoder ran with.
        `_controls` (from `_controls_for`): prosody factors (speed, pitch, energy) per phoneme, in inference only, and
        only where an utterance's result does not depend on its batch mates (per_utterance, or B = 1); the returned
        durations are then the frame counts actually expanded."""
        # the handle-less ABI stages (LengthRegulator, losses, ...) run on the CURRENT device like any CUDA library call:
        # select the device the data lives on for the whole call, leave the caller's current device untouched
        if xs.is_cuda and torch.cuda.current_device() != (xs.device.index or 0):
            with torch.cuda.device(xs.device):
                return self._forward(xs, ilens, olens, ds, es, ps, is_inference, _one_hot, _defer_check, _after_out,
                                     per_utterance, _olens_out, _controls)
        if _controls is not None:
            if not is_inference:
                raise ValueError("prosody controls apply to inference only (teacher-forced durations, energy and pitch are given)")
            if not per_utterance and xs.shape[0] != 1:
                raise ValueError("prosody controls on a batch need per_utterance=True (use synthesize): under the reference's "
                                 "batch semantics an utterance's result depends on its batch mates")
        if per_utterance:
            self._check_ilens(xs, ilens)
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
        _lib.check(lib.fs2_encode_ex(h, _lib.ptr(xs), _lib.ptr(ilens), B, T, _lib.ptr(hs), _lib.ptr(d_log), _lib.ptr(d_int),
                                     _lib.ptr(ws), ws.numel(), flags, st), "fs2_encode_ex")

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
            vals = torch.cat(words).tolist() if len(words) > 1 else stats.tolist()  # the single host sync of inference
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
        if _defer_check is not None:          # CUDA-graph capture: no host read here, the caller validates after replay
            _defer_check.append((chk_dev, T, L))
            return before, after, d_log, e_out, p_out
        if per_utterance:   # + the ilens range and olens == sum(ds) (the zero rows of hm end at sum(ds)), same transfer
            chk = torch.cat([chk_dev, torch.stack([ilens.min(), (olens_dec != olens_lr).sum()])]).tolist()
            self._check_ilens_range(chk[4], chk[2], T)
            if chk[5]:
                raise ValueError(f"per_utterance: olens differs from sum(ds) in {chk[5]} utterance(s)")
        else:
            chk = chk_dev.tolist()
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

    def forward(self, xs: torch.Tensor, ilens: torch.Tensor, ys: torch.Tensor, olens: torch.Tensor, ds: torch.Tensor,
                es: torch.Tensor, ps: torch.Tensor) -> Tuple[torch.Tensor, List[Dict[str, float]]]:
        """Loss computation (fastspeech.py:245-337). Returns (loss, report_keys).  In train mode the loss is attached to
        the autograd graph of the train path (fastspeech2_b200/train.py) so `loss.backward()` fills `.grad` of every
        parameter the reference trains; `self.dropout_masks` (a train.MaskSource) may be set to inject masks."""
        if xs.is_cuda and torch.cuda.current_device() != (xs.device.index or 0):
            with torch.cuda.device(xs.device):
                return self.forward(xs, ilens, ys, olens, ds, es, ps)
        if self.training:
            from .train import train_forward
            return train_forward(self, xs, ilens, ys, olens, ds, es, ps, masks=self.dropout_masks)
        self._ready(xs)
        lib = _lib.load()
        dev = xs.device
        ilens = ilens.to(device=dev, dtype=torch.int64)
        olens = olens.to(device=dev, dtype=torch.int64)
        tmax, lmax = torch.stack([ilens.max(), olens.max()]).tolist()
        xs = xs[:, :tmax]  # fastspeech.py:266-267
        ds_t = ds[:, :tmax].contiguous() if ds.shape[1] != tmax else ds
        es_t, ps_t = es[:, :lmax], ps[:, :lmax]
        before, after, d_outs, e_outs, p_outs = self._forward(xs, ilens, olens, ds_t, es_t, ps_t, is_inference=False)
        if ds_t is not ds and ds_t.shape == ds[:, :tmax].shape:
            ds[:, :tmax].copy_(ds_t)
        B, T = xs.shape
        L = before.shape[1]
        ys_c = ys.to(dtype=torch.float32, device=dev).contiguous()
        es_c, ps_c = es_t.to(torch.float32).contiguous(), ps_t.to(torch.float32).contiguous()
        ds_c = ds_t.contiguous()
        out7 = torch.empty((7,), dtype=torch.float32, device=dev)
        scratch = torch.empty((16,), dtype=torch.float64, device=dev)
        _lib.check(lib.fs2_masked_losses(_lib.ptr(before), _lib.ptr(after), _lib.ptr(ys_c), int(ys_c.shape[1]), _lib.ptr(d_outs),
                                         _lib.ptr(ds_c), _lib.dur_dtype(ds_c), _lib.ptr(e_outs), _lib.ptr(p_outs), _lib.ptr(es_c),
                                         _lib.ptr(ps_c), _lib.ptr(ilens.contiguous()), _lib.ptr(olens.contiguous()), B, T, L,
                                         self.odim, _lib.ptr(out7), _lib.ptr(scratch), _lib.stream_ptr(dev)), "fs2_masked_losses")
        vals = out7.tolist()
        names = ["l1_loss", "before_loss", "after_loss", "duration_loss", "energy_loss", "pitch_loss", "loss"]
        return out7[6], [{k: v} for k, v in zip(names, vals)]

    def inference(self, x: torch.Tensor) -> torch.Tensor:
        """x [T] int64 -> mel [L, odim] (fastspeech.py:339-357)."""
        ilens = torch.tensor([x.shape[0]], dtype=torch.long, device=x.device)
        _, outs, _, _, _ = self._forward(x.unsqueeze(0), ilens, is_inference=True, _one_hot=False)
        return outs[0]

    def inference_controlled(self, x: torch.Tensor, *, speed=None, pitch=None, energy=None) -> torch.Tensor:
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
        _, outs, _, _, _ = self._forward(x.unsqueeze(0), ilens, is_inference=True, _one_hot=False, _controls=controls)
        return outs[0]

    def synthesize(self, xs: torch.Tensor, ilens: torch.Tensor, *, speed=None, pitch=None,
                   energy=None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Per-utterance batched inference (not in the reference): xs [B, Tmax] int64 (0 = pad), ilens [B] with
        1 <= ilens[b] <= Tmax -> (mels [B, Lmax, odim], olens [B] int64, durations [B, Tmax] int64), all on the device.
        durations[b], olens[b] and mels[b, :olens[b]] are bit-identical to what `inference(xs[b, :ilens[b]])` computes,
        whatever else is in the batch; mels[b, olens[b]:] and durations[b, ilens[b]:] are 0.  One host read per call.
        speed / pitch / energy: prosody controls as in `inference_controlled`, each None, a number, a [B] tensor (per
        utterance) or a [B, Tmax] tensor (per phoneme; entries past ilens[b] are ignored).  Utterance b is then
        bit-identical to `inference_controlled` on it with its slice of the controls.  durations are the frame counts expanded (after speed and
        the all-zero rule): durations.sum(1) == olens."""
        if xs.dim() != 2:
            raise ValueError("xs must be [B, Tmax]")
        controls = _controls_for(int(xs.shape[0]), int(xs.shape[1]), xs.device,
                                 {"speed": speed, "pitch": pitch, "energy": energy}, ilens)
        got: list = []
        _, after, dur, _, _ = self._forward(xs, ilens, is_inference=True, _one_hot=False, per_utterance=True, _olens_out=got,
                                            _controls=controls)
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
