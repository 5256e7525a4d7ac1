"""CPU oracle of controlled inference (prosody: speed, pitch, energy), built on oracle/fs2_oracle.py.

The reference has the three knobs at module level only: `LengthRegulator.forward(xs, ds, ilens, alpha)` scales the
durations by `torch.round(ds.float() * alpha).long()` (core/duration_modeling/length_regulator.py:57-59) and
`Energy/PitchPredictor.inference(xs, alpha)` return `predictor(xs) * alpha` before bucketize
(core/variance_predictor.py:58,140-152,213-225).  Its `_forward` passes alpha = 1 to all three (fastspeech.py:192-196).
This restates that inference path with one factor per phoneme; with constant factors it is the reference's modules
wired with those alphas (tests/golden/inf_controls.npz pins it), and per phoneme each frame takes the factor of the
phoneme it was expanded from.  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F

from oracle import fs2_oracle as O


def length_regulator(xs: torch.Tensor, ds: torch.Tensor, ilens: torch.Tensor,
                     speed: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """LengthRegulator.forward with a [B, T] factor per phoneme (length_regulator.py:57-61,86-95): d' = round-half-even
    of fp32(d) * fp32(a), then the all-zero -> all-one rule on the scaled slice.  Returns (expanded [B, Lmax, C],
    durations actually used [B, T], 0 past ilens)."""
    B, T = ds.shape
    used = torch.zeros(B, T, dtype=torch.int64)
    outs: List[torch.Tensor] = []
    for b in range(B):
        n = int(ilens[b])
        d = ds[b, :n]
        d = torch.round(d.float() * speed[b, :n].float()).long() if speed is not None else d.long()
        if d.sum() == 0:
            d = torch.ones_like(d)
        if bool((d < 0).any()):
            raise RuntimeError("negative duration")
        used[b, :n] = d
        outs.append(torch.repeat_interleave(xs[b, :n], d, dim=0))
    L = max(o.size(0) for o in outs)
    return torch.stack([F.pad(o, (0, 0, 0, L - o.size(0))) for o in outs]), used


def frame_factors(f: Optional[torch.Tensor], used: torch.Tensor, ilens: torch.Tensor, L: int) -> Optional[torch.Tensor]:
    """Per-phoneme factors [B, T] -> per-frame [B, L]: repeat_interleave by the used durations, 1.0 past each length."""
    if f is None:
        return None
    out = torch.ones(used.shape[0], L)
    for b in range(used.shape[0]):
        n = int(ilens[b])
        r = torch.repeat_interleave(f[b, :n].float(), used[b, :n])
        out[b, :r.numel()] = r
    return out


def inference_path(sd: O.SD, xs: torch.Tensor, ilens: torch.Tensor, speed=None, pitch=None, energy=None, heads: int = 2):
    """FeedForwardTransformer._forward(is_inference=True) (fastspeech.py:169-243) with per-phoneme [B, T] controls
    (None = no control).  Returns (before, after, used durations, e_ids, p_ids, e_val, p_val)."""
    hs = O.encoder(sd, xs, ilens, heads)
    d_outs = O.durations_from_log(O.predictor(sd, "duration_predictor.", hs)).masked_fill(O.pad_mask(ilens), 0)
    hs, used = length_regulator(hs, d_outs, ilens, speed)
    L = hs.shape[1]
    e_val = O.predictor(sd, "energy_predictor.predictor.", hs)
    p_val = O.predictor(sd, "pitch_predictor.predictor.", hs)
    fe, fp = frame_factors(energy, used, ilens, L), frame_factors(pitch, used, ilens, L)
    if fe is not None:
        e_val = e_val * fe             # one fp32 rounding, `xs * alpha` of variance_predictor.py:58
    if fp is not None:
        p_val = p_val * fp
    e_ids = O.bucket_ids(e_val, sd["energy_predictor.energy_bins"])
    p_ids = O.bucket_ids(p_val, sd["pitch_predictor.pitch_bins"])
    hs = hs + F.linear(F.one_hot(p_ids.long(), 256).float(), sd["pitch_embed.weight"], sd["pitch_embed.bias"])
    hs = hs + F.linear(F.one_hot(e_ids.long(), 256).float(), sd["energy_embed.weight"], sd["energy_embed.bias"])
    zs = O.decoder(sd, hs, None, heads)
    odim = sd["feat_out.weight"].size(0)
    before = F.linear(zs, sd["feat_out.weight"], sd["feat_out.bias"]).view(zs.size(0), -1, odim)
    after = before + O.postnet(sd, before)
    return before, after, used, e_ids, p_ids, e_val, p_val


def per_phoneme(v, T: int) -> Optional[torch.Tensor]:
    """A scalar or [T] control -> [1, T] float32 (None stays None)."""
    if v is None:
        return None
    t = torch.as_tensor(v, dtype=torch.float32)
    return (t.expand(T) if t.dim() == 0 else t).reshape(1, T).contiguous()
