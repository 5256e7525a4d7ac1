#!/usr/bin/env python
"""Generate tests/golden/speakers.npz: the multi-speaker extension (DESIGN.md section 25) on the UNMODIFIED reference.

Run in the build container only, like make_golden.py (it imports the reference checkout):

    python tests/golden/make_golden_speakers.py

The reference has no speaker input.  Its instance's `encoder` is wrapped to return `hs + E[spk].unsqueeze(1)`, which is
what ESPnet2's and ming024's FastSpeech2 do with a speaker table, and everything downstream (duration predictor, length
regulator, variance adaptor, decoder, losses, autograd) is the reference's own code.  No reference source is modified.
Stored: the seeded inputs (a ragged B = 8 batch with repeated and distinct speakers, n_speakers = 5 of which speaker 4 is
absent, and the seeded table; the mel targets ys are not stored, `fastspeech2_b200.synthetic.make_batch(**BATCH)`
regenerates them with the rest of the batch), inference and teacher-forced outputs, and one train step's loss, report
and gradients (every parameter's largest element and a seeded sample, as train_step.npz stores them, plus the whole table
gradient) with its dropout masks drawn the way train_step.npz draws them.  The full mels would be 2.3 MB, so, as
filelist64.npz does, the fixture keeps every duration, energy, pitch and bucket id, the `after` mels of three utterances (`ROWS`:
two of one speaker, one of another), the `before` mel of the shortest, and per-utterance means over the valid frames of
every mel.  The gradient samples are stored as one array in parameter order (`grad_names`, `grad_max`, `grad_vals`);
their indices are not stored but redrawn by `sample_indices`, which the tests restate.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as G  # noqa: E402  (sets up the reference import; main() is not run)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from fastspeech import FeedForwardTransformer  # noqa: E402  (the reference)
from utils.hparams import HParam  # noqa: E402
from fastspeech2_b200.synthetic import make_batch  # noqa: E402
from fastspeech2_b200.weights import ModelDims, synthetic_state_dict  # noqa: E402

N_SPEAKERS, TABLE_SEED, TABLE_SCALE = 5, 23, 0.5
SPEAKERS = [0, 3, 3, 1, 0, 2, 3, 1]
BATCH = dict(B=8, T=19, L=120, seed=31, ilens=[19, 15, 11, 19, 7, 13, 4, 16], olens=[120, 90, 70, 110, 40, 85, 25, 100])
KEYS = ("xs", "ilens", "ys", "olens", "ds", "es", "ps")
ROWS = (2, 4, 6)            # utterances whose whole `after` mels are kept: speakers 3, 0, 3
BEFORE_ROW = 6              # and whose `before` mel is kept (the shortest)


def sample_indices(numels, seed: int = 99, k: int = G.GRAD_SAMPLES):
    """The sampled elements of each gradient: randperm(numel)[:k] from one generator, in parameter order."""
    g = torch.Generator().manual_seed(seed)
    return [torch.randperm(int(n), generator=g)[:k] for n in numels]


def mel_subset(prefix: str, before: torch.Tensor, after: torch.Tensor, olens: torch.Tensor) -> dict:
    """The mels of ROWS up to their lengths, and per-utterance means of before / after / |after| over valid frames."""
    out = {}
    for b in ROWS:
        out[f"{prefix}_after/{b}"] = after[b, :olens[b]]
    out[f"{prefix}_before/{BEFORE_ROW}"] = before[BEFORE_ROW, :olens[BEFORE_ROW]]
    valid = (torch.arange(after.shape[1])[None, :] < olens[:, None]).double()[..., None]
    n = olens.double() * after.shape[2]
    out[f"{prefix}_after_mean"] = (after.double() * valid).sum((1, 2)) / n
    out[f"{prefix}_after_absmean"] = (after.double().abs() * valid).sum((1, 2)) / n
    out[f"{prefix}_before_mean"] = (before.double() * valid).sum((1, 2)) / n
    return out


def seeded_table() -> torch.Tensor:
    return torch.randn(N_SPEAKERS, 256, generator=torch.Generator().manual_seed(TABLE_SEED)) * TABLE_SCALE


def with_speakers(ref, table: torch.Tensor, spk: torch.Tensor):
    """Wrap the instance's encoder: (hs, masks) -> (hs + table[spk].unsqueeze(1), masks)."""
    inner = ref.encoder.forward

    def forward(xs, masks):
        hs, m = inner(xs, masks)
        return hs + table[spk].unsqueeze(1), m
    ref.encoder.forward = forward
    return ref


def main():
    torch.set_num_threads(1)
    bt = make_batch(BATCH["B"], BATCH["T"], BATCH["L"], seed=BATCH["seed"], ilens=BATCH["ilens"], olens=BATCH["olens"])
    spk = torch.tensor(SPEAKERS, dtype=torch.int64)
    table = seeded_table()
    out = {k: bt[k] for k in KEYS if k != "ys"}
    out.update(speakers=spk, table=table, n_speakers=np.int64(N_SPEAKERS), batch=json.dumps(BATCH))

    model, _ = G.build_reference()
    with_speakers(model, table, spk)
    with torch.no_grad():
        b, a, d, e, p = model._forward(bt["xs"], bt["ilens"], bt["olens"], bt["ds"].clone(), bt["es"], bt["ps"], is_inference=False)
        out.update(tf_d_outs=d, tf_e_outs=e, tf_p_outs=p, **mel_subset("tf", b, a, bt["olens"]))
        b, a, d, eh, ph = model._forward(bt["xs"], bt["ilens"], is_inference=True)
        out.update(inf_d_outs=d, inf_e_ids=eh.argmax(-1).to(torch.int16), inf_p_ids=ph.argmax(-1).to(torch.int16),
                   inf_frames=np.int64(a.shape[1]), **mel_subset("inf", b, a, d.sum(1)))

    # one train step, masks from torch.rand(shape, generator seeded 5) >= p in call order (make_golden.train_step_fixture)
    torch.manual_seed(0)
    ref = FeedForwardTransformer(68, 80, HParam("configs/default.yaml"))
    ref.load_state_dict(synthetic_state_dict(G.WEIGHT_SEED, ModelDims()), strict=True)
    ref.train()
    tab = table.clone().requires_grad_()
    with_speakers(ref, tab, spk)
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
    idx = sample_indices([g.numel() for _, g in named])
    out["no_grad"] = json.dumps([n for n, p in ref.named_parameters() if p.grad is None])
    out["grad_names"] = json.dumps([n for n, _ in named])
    out["grad_max"] = torch.stack([g.abs().max() for _, g in named])
    out["grad_vals"] = torch.cat([g[i] for (_, g), i in zip(named, idx)])
    out["grad/speaker_embed.weight"] = tab.grad.detach()
    for bname, buf in ref.named_buffers():
        if "running" in bname or "num_batches" in bname:
            out["buf/" + bname] = buf.detach()
    G.npz("speakers", **out)


if __name__ == "__main__":
    main()
