"""CPU oracle of the external speaker embeddings (DESIGN.md section 27).

TEST INFRASTRUCTURE ONLY, like fs2_oracle.py, whose functions it reuses unchanged.  The only new step is ESPnet2's
`spembs` add (integration type "add"): `hs + E[spk].unsqueeze(1) + proj(F.normalize(spembs)).unsqueeze(1)` after the
encoder, the table optional.  Pinned by tests/test_spembs_args.py against tests/golden/spembs.npz, which
tests/golden/make_golden_spembs.py writes from the unmodified reference with its encoder wrapped the same way.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.nn.functional as F

from . import fs2_oracle as O


def project(W: torch.Tensor, bias: torch.Tensor, spembs: torch.Tensor) -> torch.Tensor:
    """v = W . normalize(spembs) + bias, [B, adim]."""
    return F.linear(F.normalize(spembs), W, bias)


def forward_path(sd: O.SD, table: Optional[torch.Tensor], speakers: Optional[torch.Tensor], W: torch.Tensor, bias: torch.Tensor,
                 spembs: torch.Tensor, xs: torch.Tensor, ilens: torch.Tensor, olens: Optional[torch.Tensor] = None,
                 ds: Optional[torch.Tensor] = None, es: Optional[torch.Tensor] = None, ps: Optional[torch.Tensor] = None,
                 is_inference: bool = False, heads: int = 2) -> Tuple[torch.Tensor, ...]:
    """fs2_oracle.forward_path with (hs [+ table[speakers]]) + v after the encoder."""
    hs = O.encoder(sd, xs, ilens, heads)
    if table is not None:
        hs = hs + table[speakers].unsqueeze(1)
    hs = hs + project(W, bias, spembs).unsqueeze(1)
    d_masks = O.pad_mask(ilens)
    e_bins, p_bins = sd["energy_predictor.energy_bins"], sd["pitch_predictor.pitch_bins"]
    if is_inference:
        d_outs = O.durations_from_log(O.predictor(sd, "duration_predictor.", hs)).masked_fill(d_masks, 0)
        hs = O.length_regulator(hs, d_outs, ilens)
        e_ids = O.bucket_ids(O.predictor(sd, "energy_predictor.predictor.", hs), e_bins)
        p_ids = O.bucket_ids(O.predictor(sd, "pitch_predictor.predictor.", hs), p_bins)
        e_ret, p_ret = F.one_hot(e_ids.long(), 256).float(), F.one_hot(p_ids.long(), 256).float()
    else:
        e_ids, p_ids = O.bucket_ids(es, e_bins), O.bucket_ids(ps, p_bins)
        mel_masks = O.pad_mask(olens)
        d_outs = O.predictor(sd, "duration_predictor.", hs).masked_fill(d_masks, 0.0)
        hs = O.length_regulator(hs, ds, ilens)
        e_ret = O.predictor(sd, "energy_predictor.predictor.", hs).masked_fill(mel_masks, 0.0)
        p_ret = O.predictor(sd, "pitch_predictor.predictor.", hs).masked_fill(mel_masks, 0.0)
    hs = hs + F.linear(F.one_hot(p_ids.long(), 256).float(), sd["pitch_embed.weight"], sd["pitch_embed.bias"])
    hs = hs + F.linear(F.one_hot(e_ids.long(), 256).float(), sd["energy_embed.weight"], sd["energy_embed.bias"])
    zs = O.decoder(sd, hs, olens, heads)
    odim = sd["feat_out.weight"].size(0)
    before = F.linear(zs, sd["feat_out.weight"], sd["feat_out.bias"]).view(zs.size(0), -1, odim)
    after = before + O.postnet(sd, before)
    return before, after, d_outs, e_ret, p_ret
