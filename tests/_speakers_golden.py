"""Reading tests/golden/speakers.npz (tests/golden/make_golden_speakers.py), shared by the CPU and GPU speaker tests."""
import json

import numpy as np
import torch

from fastspeech2_b200.synthetic import make_batch

ROWS, BEFORE_ROW, GRAD_SAMPLES = (2, 4, 6), 6, 96      # as make_golden_speakers.py stores them


def batch(g) -> dict:
    """The fixture's batch on the host: make_batch(**batch) regenerates ys; the stored inputs must agree with it."""
    c = json.loads(str(g["batch"]))
    bt = make_batch(c["B"], c["T"], c["L"], seed=c["seed"], ilens=c["ilens"], olens=c["olens"])
    for k in ("xs", "ilens", "olens", "ds", "es", "ps"):
        assert np.array_equal(bt[k].numpy(), g[k]), k
    return bt


def sample_indices(numels, seed: int = 99, k: int = GRAD_SAMPLES):
    """make_golden_speakers.sample_indices: randperm(numel)[:k] from one generator, in parameter order."""
    gen = torch.Generator().manual_seed(seed)
    return [torch.randperm(int(n), generator=gen)[:k] for n in numels]


def grad_samples(g, numels: dict) -> dict:
    """{name: (indices, reference values, reference max |grad|)} for every parameter the reference has a gradient for;
    numels maps each name to its element count."""
    names = json.loads(str(g["grad_names"]))
    idx = sample_indices([numels[n] for n in names])
    vals, out, o = torch.from_numpy(g["grad_vals"]), {}, 0
    for n, i, m in zip(names, idx, g["grad_max"].tolist()):
        out[n] = (i, vals[o: o + len(i)], m)
        o += len(i)
    assert o == vals.numel()
    return out


def mel_checks(g, prefix: str, before: torch.Tensor, after: torch.Tensor, olens: torch.Tensor):
    """(what, got, want) pairs: the kept mels up to their lengths, and per-utterance means over the valid frames."""
    before, after, olens = before.double().cpu(), after.double().cpu(), olens.cpu()
    out = [(f"after[{b}]", after[b, :olens[b]], g[f"{prefix}_after/{b}"]) for b in ROWS]
    out.append((f"before[{BEFORE_ROW}]", before[BEFORE_ROW, :olens[BEFORE_ROW]], g[f"{prefix}_before/{BEFORE_ROW}"]))
    valid = (torch.arange(after.shape[1])[None, :] < olens[:, None]).double()[..., None]
    n = olens.double() * after.shape[2]
    return out, [("after means", (after * valid).sum((1, 2)) / n, g[f"{prefix}_after_mean"]),
                 ("after abs means", (after.abs() * valid).sum((1, 2)) / n, g[f"{prefix}_after_absmean"]),
                 ("before means", (before * valid).sum((1, 2)) / n, g[f"{prefix}_before_mean"])]
