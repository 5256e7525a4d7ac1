#!/usr/bin/env python
"""Generate tests/golden/inf_controls.npz from the UNMODIFIED reference (build container only, like make_golden.py,
whose import shim and checkpoint this reuses):

    python tests/golden/make_golden_controls.py

The reference's inference `_forward` (fastspeech.py:169-243) is wired by hand with its own modules and scalar alphas
passed to `length_regulator(hs, d_outs, ilens, alpha)` and `energy/pitch_predictor.inference(hs, alpha)`
(length_regulator.py:57-59, variance_predictor.py:58,140-152,213-225), which `_forward` calls with alpha = 1.  B = 1.
The cases cover a factor fp32 cannot represent (1.1), semitone factors, and a speed that lands on half-way ties (2.5).
The LengthRegulator cases pin the duration rule itself on ties and on the all-zero -> all-one rule after scaling.
Only inputs and outputs are stored."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports the reference through its shim; chdir to the checkout)

import torch  # noqa: E402

from utils.util import make_pad_mask  # noqa: E402  (the reference)

CASES = [(1.1, 2 ** (3 / 12), 1.1), (2.5, 2 ** (-5 / 12), 0.8), (0.75, 1.1, 1.25)]   # (speed, pitch, energy)
LR_ALPHAS = [2.5, 3.5, 0.4, 1.1]


def controlled_inference(model, x, speed, pitch, energy):
    xs, ilens = x.unsqueeze(0), torch.tensor([x.shape[0]])
    hs, _ = model.encoder(xs, model._source_mask(ilens))
    d_outs = model.duration_predictor.inference(hs, make_pad_mask(ilens))
    hs = model.length_regulator(hs, d_outs, ilens, speed)
    e_val = model.energy_predictor.predictor.inference(hs, False, alpha=energy)
    p_val = model.pitch_predictor.predictor.inference(hs, False, alpha=pitch)
    one_hot_energy = model.energy_predictor.inference(hs, energy)
    one_hot_pitch = model.pitch_predictor.inference(hs, pitch)
    hs = hs + model.pitch_embed(one_hot_pitch)
    hs = hs + model.energy_embed(one_hot_energy)
    zs, _ = model.decoder(hs, None)
    before = model.feat_out(zs).view(zs.size(0), -1, model.odim)
    after = before + model.postnet(before.transpose(1, 2)).transpose(1, 2)
    return before, after, d_outs, one_hot_energy.argmax(-1), one_hot_pitch.argmax(-1), e_val, p_val


def main():
    model, _ = G.build_reference()
    x = torch.randint(1, 68, (23,), generator=torch.Generator().manual_seed(13))   # inf_single's utterance
    out = {"x": x, "cases": torch.tensor(CASES, dtype=torch.float64)}
    with torch.no_grad():
        for i, (s, p, e) in enumerate(CASES):
            b, a, d, ei, pi, ev, pv = controlled_inference(model, x, s, p, e)
            out.update({f"mel{i}": a[0], f"d_pred{i}": d[0], f"e_ids{i}": ei[0], f"p_ids{i}": pi[0],
                        f"e_val{i}": ev[0], f"p_val{i}": pv[0]})
    lr = G.LengthRegulator()
    g = torch.Generator().manual_seed(18)
    hs = torch.randn(3, 8, 4, generator=g)
    il = torch.tensor([8, 5, 3])
    d = torch.tensor([[1, 3, 5, 7, 2, 0, 4, 6],      # odd x 2.5 and x 3.5 land on ties
                      [1, 1, 1, 1, 1, 9, 9, 9],      # x 0.4: all round to 0 -> filled with 1 (past ilen ignored)
                      [0, 1, 2, 0, 0, 0, 0, 0]])
    out.update({"lr_hs": hs, "lr_ilens": il, "lr_d": d, "lr_alphas": torch.tensor(LR_ALPHAS, dtype=torch.float64)})
    for i, alpha in enumerate(LR_ALPHAS):
        out[f"lr_out{i}"] = lr(hs, d.clone(), il, alpha)
    G.npz("inf_controls", **out)


if __name__ == "__main__":
    main()
