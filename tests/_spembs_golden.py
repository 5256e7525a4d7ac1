"""Reading tests/golden/spembs.npz (tests/golden/make_golden_spembs.py), shared by the CPU and GPU speaker-embedding tests.
The batch, the gradient samples and the per-utterance mel checks are those of speakers.npz (tests/_speakers_golden.py);
the embeddings and the projection are regenerated here from make_golden_spembs.py's seeds."""
import torch

import _speakers_golden as SG

D, SEED = 192, 41
CONFIGS = ("both", "emb")           # the speaker table and the embeddings together; the embeddings alone
batch, grad_samples = SG.batch, SG.grad_samples


def seeded(B: int = 8):
    """make_golden_spembs.seeded: (spembs [B, D], W [256, D], bias [256])."""
    g = torch.Generator().manual_seed(SEED)
    e = torch.randn(B, D, generator=g) * 3.0
    e[3] = 0.0
    e[5] = e[1]
    W = torch.randn(256, D, generator=g) * 0.5
    bias = torch.randn(256, generator=g) * 0.1
    return e, W, bias


def table() -> torch.Tensor:
    """make_golden_speakers.seeded_table: the speaker table [5, 256]."""
    return torch.randn(5, 256, generator=torch.Generator().manual_seed(23)) * 0.5


def cfg(g, name: str) -> dict:
    """The entries of one configuration without their prefix, in the key layout of speakers.npz."""
    p = name + "/"
    return {k[len(p):]: v for k, v in g.items() if k.startswith(p)}


def mel_checks(g, prefix: str, before, after, olens):
    return SG.mel_checks(g, prefix, before, after, olens)
