#!/usr/bin/env python
"""Generate tests/golden/spembs.npz: external speaker embeddings (DESIGN.md section 27) on the UNMODIFIED reference.

Run in the build container only, like make_golden.py (it imports the reference checkout):

    python tests/golden/make_golden_spembs.py

The reference takes no speaker input.  As make_golden_speakers.py does for the table, its instance's `encoder` is wrapped to
return `hs + E[spk].unsqueeze(1) + proj(F.normalize(spembs)).unsqueeze(1)`, which is ESPnet2's FastSpeech2 with a speaker
table and `spk_embed_integration_type = "add"`; everything downstream is the reference's own code.  No reference source is
modified.  Two configurations on the ragged B = 8 batch of speakers.npz, with D = 192:
  "both": the speaker table and the embeddings together;   "emb": the embeddings alone.
Utterance 3's embedding is all zeros (normalize leaves it 0, so only the bias is added), and utterances 1 and 5 share one.
Stored per configuration, as speakers.npz stores them: inference and teacher-forced durations, energies, pitches and
bucket ids, three utterances' `after` mels, one `before` mel and per-utterance means of every mel.  For "both", one train
step: loss, report, each gradient's largest element and a seeded sample (in the order of fastspeech2_b200's parameters:
the reference's, then speaker_embed.weight, spk_embed_proj.weight and .bias), and the whole table and bias gradients.  The
mel targets, the embeddings, the table and the projection are regenerated from their seeds (tests/_spembs_golden.py).
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as G  # noqa: E402  (sets up the reference import; main() is not run)
import make_golden_speakers as GS  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from fastspeech import FeedForwardTransformer  # noqa: E402  (the reference)
from utils.hparams import HParam  # noqa: E402
from fastspeech2_b200.synthetic import make_batch  # noqa: E402
from fastspeech2_b200.weights import ModelDims, synthetic_state_dict  # noqa: E402

D, SEED = 192, 41
KEYS = GS.KEYS


def seeded(B: int = 8):
    """(spembs [B, D], W [256, D], bias [256]): x-vector-like embeddings of norm ~40, utterance 3 all zeros, utterances 1
    and 5 equal; a projection whose output has a standard deviation of about 0.5."""
    g = torch.Generator().manual_seed(SEED)
    e = torch.randn(B, D, generator=g) * 3.0
    e[3] = 0.0
    e[5] = e[1]
    W = torch.randn(256, D, generator=g) * 0.5
    bias = torch.randn(256, generator=g) * 0.1
    return e, W, bias


def with_spembs(ref, table, spk, W, bias, e):
    """Wrap the instance's encoder: (hs, masks) -> (hs [+ table[spk]] + (normalize(e) W^T + bias), masks)."""
    inner = ref.encoder.forward

    def forward(xs, masks):
        hs, m = inner(xs, masks)
        if table is not None:
            hs = hs + table[spk].unsqueeze(1)
        return hs + F.linear(F.normalize(e), W, bias).unsqueeze(1), m
    ref.encoder.forward = forward
    return ref


def main():
    torch.set_num_threads(1)
    c = GS.BATCH
    bt = make_batch(c["B"], c["T"], c["L"], seed=c["seed"], ilens=c["ilens"], olens=c["olens"])
    spk = torch.tensor(GS.SPEAKERS, dtype=torch.int64)
    table = GS.seeded_table()
    e, W, bias = seeded()
    out = {k: bt[k] for k in KEYS if k != "ys"}
    out.update(speakers=spk, n_speakers=np.int64(GS.N_SPEAKERS), D=np.int64(D), batch=json.dumps(GS.BATCH))

    for cfg, tab in (("both", table), ("emb", None)):
        model, _ = G.build_reference()
        with_spembs(model, tab, spk, W, bias, e)
        with torch.no_grad():
            b, a, d, eo, po = model._forward(bt["xs"], bt["ilens"], bt["olens"], bt["ds"].clone(), bt["es"], bt["ps"],
                                             is_inference=False)
            out.update({f"{cfg}/tf_d_outs": d, f"{cfg}/tf_e_outs": eo, f"{cfg}/tf_p_outs": po})
            out.update({f"{cfg}/{k}": v for k, v in GS.mel_subset("tf", b, a, bt["olens"]).items()})
            b, a, d, eh, ph = model._forward(bt["xs"], bt["ilens"], is_inference=True)
            out.update({f"{cfg}/inf_d_outs": d, f"{cfg}/inf_e_ids": eh.argmax(-1).to(torch.int16),
                        f"{cfg}/inf_p_ids": ph.argmax(-1).to(torch.int16), f"{cfg}/inf_frames": np.int64(a.shape[1])})
            out.update({f"{cfg}/{k}": v for k, v in GS.mel_subset("inf", b, a, d.sum(1)).items()})

    # one train step of "both", masks as in make_golden_speakers.py
    torch.manual_seed(0)
    ref = FeedForwardTransformer(68, 80, HParam("configs/default.yaml"))
    ref.load_state_dict(synthetic_state_dict(G.WEIGHT_SEED, ModelDims()), strict=True)
    ref.train()
    tab = table.clone().requires_grad_()
    Wg, bg = W.clone().requires_grad_(), bias.clone().requires_grad_()
    with_spembs(ref, tab, spk, Wg, bg, e)
    gen = torch.Generator().manual_seed(5)
    shapes, rates = [], []
    real = torch.nn.functional.dropout

    def shared_dropout(input, p=0.5, training=True, inplace=False):
        if not training or p == 0.0:
            return input
        m = torch.rand(input.shape, generator=gen) >= p
        shapes.append(list(input.shape)); rates.append(p)
        return input * m.to(input.dtype) / (1.0 - p)

    torch.nn.functional.dropout = shared_dropout
    try:
        loss, rep = ref(*[bt[k] for k in KEYS])
        loss.backward()
    finally:
        torch.nn.functional.dropout = real
    out.update({"mask_shapes": json.dumps(shapes), "mask_rates": np.array(rates, dtype=np.float64), "loss": float(loss.detach()),
                "report_names": json.dumps([list(r)[0] for r in rep]),
                "report_values": np.array([float(list(r.values())[0]) for r in rep], dtype=np.float64)})
    named = [(n, p.grad.detach().reshape(-1)) for n, p in ref.named_parameters() if p.grad is not None]
    named += [("speaker_embed.weight", tab.grad.reshape(-1)), ("spk_embed_proj.weight", Wg.grad.reshape(-1)),
              ("spk_embed_proj.bias", bg.grad.reshape(-1))]
    idx = GS.sample_indices([g.numel() for _, g in named])
    out["no_grad"] = json.dumps([n for n, p in ref.named_parameters() if p.grad is None])
    out["grad_names"] = json.dumps([n for n, _ in named])
    out["grad_max"] = torch.stack([g.abs().max() for _, g in named])
    out["grad_vals"] = torch.cat([g[i] for (_, g), i in zip(named, idx)])
    out["grad/speaker_embed.weight"] = tab.grad.detach()
    out["grad/spk_embed_proj.bias"] = bg.grad.detach()
    G.npz("spembs", **out)


if __name__ == "__main__":
    main()
