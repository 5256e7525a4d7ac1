"""TorchScript / serving variant (SURVEY.md section 8f-4): what the reference ships as `utils/fastspeech2_script.py`
(a scriptable re-statement of the model whose `forward(x [T]) -> mel [L, odim]`, :201-219) plus `export_torchscript.py`
(:35-59: `torch.jit.script(model).save(...)`, optionally `torch.jit.trace`).

Here the exported module does not re-state the network in TorchScript: it carries the 225 checkpoint tensors as one flat
buffer (+ their keys and shapes) and its `forward` is ONE call of the custom operator `fs2_b200::inference`, whose implementation drives the same
`libfs2b200.so` stages as `FeedForwardTransformer.inference`.  So a served `.pt` runs on the same kernels as everything else:

    from fastspeech2_b200.serving import export_torchscript          # registers torch.ops.fs2_b200.*
    export_torchscript(model, "fs2.pt")                              # export_torchscript.py:46-48
    served = torch.jit.load("fs2.pt").cuda()                         # any process that imported this module
    mel = served(torch.tensor(ids).cuda())                           # [L, odim]; batched: served.batch(xs, ilens)
    mels, olens = served.synthesize(xs, ilens)                       # batched, each utterance independent of its batch mates
    mels, olens, durations = served.synthesize_controlled(xs, ilens, speed, pitch, energy)   # + prosody controls
    audio, alens = served.synthesize_audio(xs, ilens, speed, pitch, energy, 30, 0.0, 0)      # + Griffin-Lim vocoder

The operator is registered through `torch.library` (schema + CUDA implementation); there is no CPU implementation -- a
CPU tensor fails loudly like the rest of the path.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Tuple

import torch

from .fastspeech import FeedForwardTransformer
from .hparams import load_hp
from .vocoder import GriffinLimVocoder

_LIB = torch.library.Library("fs2_b200", "DEF")
_LIB.define("inference(Tensor blob, str[] keys, int[] ranks, int[] dims, str precision, Tensor x) -> Tensor")
_LIB.define("inference_batch(Tensor blob, str[] keys, int[] ranks, int[] dims, str precision, Tensor xs, Tensor ilens) -> (Tensor, Tensor)")
_LIB.define("synthesize_batch(Tensor blob, str[] keys, int[] ranks, int[] dims, str precision, Tensor xs, Tensor ilens) -> (Tensor, Tensor)")
_LIB.define("synthesize_controlled(Tensor blob, str[] keys, int[] ranks, int[] dims, str precision, Tensor xs, Tensor ilens, "
            "Tensor speed, Tensor pitch, Tensor energy) -> (Tensor, Tensor, Tensor)")
_LIB.define("synthesize_audio(Tensor blob, str[] keys, int[] ranks, int[] dims, str precision, Tensor xs, Tensor ilens, "
            "Tensor speed, Tensor pitch, Tensor energy, int n_iters, float momentum, int seed) -> (Tensor, Tensor)")

# one packed model per (device, identity of the checkpoint blob): the op is functional from TorchScript's point of view,
# the cache only avoids re-packing the checkpoint on every call
_MODELS: Dict[Tuple, FeedForwardTransformer] = {}
_VOCODERS: Dict[str, GriffinLimVocoder] = {}     # math mode -> vocoder with the default config's audio parameters


def pack_state(state_dict: Dict[str, torch.Tensor]):
    """Checkpoint -> (one flat fp32 blob, keys, ranks, flattened dims).  TorchScript modules cannot hold a dynamic list of
    buffers, so the 225 tensors travel as one buffer plus their shapes; integer tensors (BatchNorm's
    num_batches_tracked, unused by the forward path) are stored as fp32 and restored as int64."""
    keys, ranks, dims, parts = [], [], [], []
    for k, v in state_dict.items():
        keys.append(k); ranks.append(v.dim()); dims.extend(int(d) for d in v.shape)
        parts.append(v.detach().reshape(-1).to(torch.float32))
    return torch.cat(parts), keys, ranks, dims


def unpack_state(blob: torch.Tensor, keys: List[str], ranks: List[int], dims: List[int]) -> Dict[str, torch.Tensor]:
    sd, off, di = {}, 0, 0
    for k, r in zip(keys, ranks):
        shape = [int(d) for d in dims[di: di + r]]
        di += r
        n = 1
        for d in shape:
            n *= d
        t = blob[off: off + n].view(shape)
        off += n
        sd[k] = t.to(torch.int64) if k.endswith("num_batches_tracked") else t
    return sd


def _model_for(blob: torch.Tensor, keys: List[str], ranks: List[int], dims: List[int], precision: str) -> FeedForwardTransformer:
    ident = (str(blob.device), precision, blob.data_ptr(), blob._version, blob.numel())
    m = _MODELS.get(ident)
    if m is None:
        if len(_MODELS) > 8:
            _MODELS.clear()
        sd = unpack_state(blob, keys, ranks, dims)
        idim, odim = int(sd["encoder.embed.0.weight"].shape[0]), int(sd["feat_out.weight"].shape[0])
        m = FeedForwardTransformer(idim, odim, load_hp(), precision=precision or None)
        m.load_state_dict(sd, strict=True)
        m = m.to(blob.device).eval()
        _MODELS[ident] = m
    return m


def _inference(blob, keys, ranks, dims, precision, x):
    with torch.no_grad():
        return _model_for(blob, keys, ranks, dims, precision).inference(x)


def _inference_batch(blob, keys, ranks, dims, precision, xs, ilens):
    with torch.no_grad():
        _, after, d, _, _ = _model_for(blob, keys, ranks, dims, precision)._forward(xs, ilens, is_inference=True, _one_hot=False)
    return after, d.sum(dim=1)


def _synthesize_batch(blob, keys, ranks, dims, precision, xs, ilens):
    with torch.no_grad():
        mels, olens, _ = _model_for(blob, keys, ranks, dims, precision).synthesize(xs, ilens)
    return mels, olens


def _synthesize_controlled(blob, keys, ranks, dims, precision, xs, ilens, speed, pitch, energy):
    with torch.no_grad():
        return _model_for(blob, keys, ranks, dims, precision).synthesize(xs, ilens, speed=speed, pitch=pitch, energy=energy)


def _synthesize_audio(blob, keys, ranks, dims, precision, xs, ilens, speed, pitch, energy, n_iters, momentum, seed):
    m = _model_for(blob, keys, ranks, dims, precision)
    voc = _VOCODERS.get(m.precision)
    if voc is None:
        voc = _VOCODERS[m.precision] = GriffinLimVocoder.from_hp(load_hp(), math_mode=m.precision)
    with torch.no_grad():
        mels, olens, _ = m.synthesize(xs, ilens, speed=speed, pitch=pitch, energy=energy)
        return voc(mels, olens, n_iters=n_iters, momentum=momentum, seed=seed)


def _no_cpu(*a, **k):
    raise RuntimeError("fs2_b200 operators run on CUDA tensors only (the H100 path has no CPU fallback)")


_LIB.impl("inference", _inference, "CUDA")
_LIB.impl("inference_batch", _inference_batch, "CUDA")
_LIB.impl("synthesize_batch", _synthesize_batch, "CUDA")
_LIB.impl("synthesize_controlled", _synthesize_controlled, "CUDA")
_LIB.impl("synthesize_audio", _synthesize_audio, "CUDA")
_LIB.impl("inference", _no_cpu, "CPU")
_LIB.impl("inference_batch", _no_cpu, "CPU")
_LIB.impl("synthesize_batch", _no_cpu, "CPU")
_LIB.impl("synthesize_controlled", _no_cpu, "CPU")
_LIB.impl("synthesize_audio", _no_cpu, "CPU")


class ScriptedFastSpeech2(torch.nn.Module):
    """Scriptable serving module: one buffer = the reference checkpoint, forward = the custom operator."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], precision: str = ""):
        super().__init__()
        blob, keys, ranks, dims = pack_state(state_dict)
        self.register_buffer("blob", blob)
        self.keys: List[str] = keys
        self.ranks: List[int] = ranks
        self.dims: List[int] = dims
        self.precision: str = precision

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x [T] int64 -> mel [L, odim]  (utils/fastspeech2_script.py:201-219)."""
        return torch.ops.fs2_b200.inference(self.blob, self.keys, self.ranks, self.dims, self.precision, x)

    @torch.jit.export
    def batch(self, xs: torch.Tensor, ilens: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """xs [B,T] int64 (0 = pad), ilens [B] -> (mels [B,Lmax,odim], olens [B])."""
        return torch.ops.fs2_b200.inference_batch(self.blob, self.keys, self.ranks, self.dims, self.precision, xs, ilens)

    @torch.jit.export
    def synthesize(self, xs: torch.Tensor, ilens: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """Per-utterance batch for dynamic batching: xs [B,T] int64 (0 = pad), ilens [B] -> (mels [B,Lmax,odim], olens [B]).
        Each utterance's mels are bit-identical to forward() on it alone, whatever else is in the batch; padded frames
        are 0 (FeedForwardTransformer.synthesize)."""
        return torch.ops.fs2_b200.synthesize_batch(self.blob, self.keys, self.ranks, self.dims, self.precision, xs, ilens)

    @torch.jit.export
    def synthesize_controlled(self, xs: torch.Tensor, ilens: torch.Tensor, speed: torch.Tensor, pitch: torch.Tensor,
                              energy: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """`synthesize` with prosody controls (e.g. SSML <prosody rate= pitch= volume=>): speed, pitch and energy are
        0-d tensors (one factor for the batch), [B] (per utterance) or [B, T] (per phoneme) factors, finite and > 0;
        pass torch.ones(()) for no change -> (mels [B,Lmax,odim], olens [B], durations [B,T] frame counts expanded).
        Equal to FeedForwardTransformer.synthesize with the same controls."""
        return torch.ops.fs2_b200.synthesize_controlled(self.blob, self.keys, self.ranks, self.dims, self.precision, xs,
                                                        ilens, speed, pitch, energy)

    @torch.jit.export
    def synthesize_audio(self, xs: torch.Tensor, ilens: torch.Tensor, speed: torch.Tensor, pitch: torch.Tensor,
                         energy: torch.Tensor, n_iters: int = 30, momentum: float = 0.0,
                         seed: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
        """`synthesize_controlled` followed by the Griffin-Lim vocoder (GriffinLimVocoder with the default config's audio
        parameters, in this module's precision) -> (audio [B, (Lmax-1)*hop] fp32, alens [B] int64).  Each utterance's
        audio is independent of its batch mates; audio past alens[b] is 0."""
        return torch.ops.fs2_b200.synthesize_audio(self.blob, self.keys, self.ranks, self.dims, self.precision, xs, ilens,
                                                   speed, pitch, energy, n_iters, momentum, seed)


def scripted(model: FeedForwardTransformer, precision: Optional[str] = None) -> torch.jit.ScriptModule:
    """`torch.jit.script` of the serving wrapper around `model`'s checkpoint (export_torchscript.py:46-47)."""
    wrapper = ScriptedFastSpeech2(model.state_dict(), precision if precision is not None else model.precision)
    return torch.jit.script(wrapper)


def export_torchscript(model: FeedForwardTransformer, path: str, precision: Optional[str] = None) -> str:
    """export_torchscript.py:46-48: script + save.  Load with `torch.jit.load(path)` in a process that has imported
    `fastspeech2_b200.serving` (which registers the operator and locates libfs2b200.so)."""
    m = scripted(model, precision)
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    m.save(path)
    return path
