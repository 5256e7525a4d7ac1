"""Float64 restatement of the duration aligner (fastspeech2_b200/aligner.py, DESIGN.md section 24): the model, the
beta-binomial prior, the forward-sum and binarization losses in numpy / CPU torch, plus the float32 MAS the kernel must
match bit for bit.

TEST INFRASTRUCTURE ONLY.  Layouts are the kernels': xs [B, T] int64, mels [B, L, 80], q [B, L, 80], k [B, T, 80],
logp [B, L, T].  State dicts are `Aligner.state_dict()`."""
from __future__ import annotations

import numpy as np
import scipy.stats
import torch
import torch.nn.functional as F

TEMP = 0.0005


def prior(N: int, M: int) -> np.ndarray:
    """[M, N] float64: betabinom(N, l + 1, M - l).pmf(t) for frames l < M and phonemes t < N (FastPitch's prior)."""
    t = np.arange(N)
    return np.stack([scipy.stats.betabinom(N, l + 1, M - l).pmf(t) for l in range(M)])


def log_prior(N: int, M: int) -> np.ndarray:
    """[M, N] float32: log(prior + 1e-8) in float64, rounded once, as the kernel adds it."""
    return np.log(prior(N, M) + 1e-8).astype(np.float32)


def _mask(x: torch.Tensor, lens) -> torch.Tensor:
    """x [B, L, C] with rows t >= lens[b] set to 0."""
    keep = torch.arange(x.shape[1])[None, :] < torch.as_tensor(lens)[:, None]
    return x * keep[:, :, None].to(x.dtype)


def _conv(x: torch.Tensor, lens, w, b, relu: bool) -> torch.Tensor:
    y = F.conv1d(_mask(x, lens).transpose(1, 2), w, b, padding=(w.shape[2] - 1) // 2).transpose(1, 2)
    return torch.relu(y) if relu else y


def keys_queries(sd: dict, xs, ilens, mels, olens):
    """(k [B, T, 80], q [B, L, 80]) in float64 (padding rows as the convolutions leave them)."""
    p = {n: v.double().cpu() for n, v in sd.items()}
    ilens, olens = torch.as_tensor(ilens).cpu(), torch.as_tensor(olens).cpu()
    h = p["embed.weight"][torch.as_tensor(xs).cpu().long()]
    h = _conv(h, ilens, p["key_conv1.weight"], p["key_conv1.bias"], True)
    k = _conv(h, ilens, p["key_conv2.weight"], p["key_conv2.bias"], False)
    m = torch.as_tensor(mels).double().cpu()
    m = _conv(m, olens, p["query_conv1.weight"], p["query_conv1.bias"], True)
    m = _conv(m, olens, p["query_conv2.weight"], p["query_conv2.bias"], True)
    q = _conv(m, olens, p["query_conv3.weight"], p["query_conv3.bias"], False)
    return k, q


def logprob(q: torch.Tensor, k: torch.Tensor, ilens, olens) -> torch.Tensor:
    """logp [B, L, T] (float64, differentiable in q and k): masked log-softmax of -0.0005 |q - k|^2 plus the log prior
    (float32, as the kernel adds it); 0 outside l < olens, t < ilens."""
    B, L, T = q.shape[0], q.shape[1], k.shape[1]
    rows = []
    for b in range(B):
        N, M = int(ilens[b]), int(olens[b])
        d = ((q[b, :M, None, :] - k[b, None, :N, :]) ** 2).sum(-1)
        lp = torch.log_softmax(-TEMP * d, dim=1) + torch.from_numpy(log_prior(N, M)).double()
        rows.append(F.pad(lp, (0, T - N, 0, L - M)))
    return torch.stack(rows)


def forward_sum(logp: torch.Tensor, ilens, olens) -> torch.Tensor:
    """[B] float64: torch ctc_loss(reduction="mean", zero_infinity=True) of the labels 1..N on log_softmax([-1, logp]) of
    each utterance alone (0 for an infeasible one)."""
    out = []
    for b in range(logp.shape[0]):
        N, M = int(ilens[b]), int(olens[b])
        if M < N:
            out.append(logp.new_zeros(()))
            continue
        z = F.pad(logp[b, :M, :N], (1, 0), value=-1.0)
        lp = torch.log_softmax(z, dim=1)[:, None, :]
        out.append(F.ctc_loss(lp, torch.arange(1, N + 1)[None], torch.tensor([M]), torch.tensor([N]), blank=0,
                              reduction="mean", zero_infinity=True))
    return torch.stack(out)


def ctc_direct(lp: np.ndarray) -> float:
    """CTC negative log-likelihood of the labels 1..N over the frames of lp [M, N + 1] (column 0 the blank), summed over
    every monotonic path of the blank-extended label sequence in probability space (float64, no logs in the lattice)."""
    M, N = lp.shape[0], lp.shape[1] - 1
    S = 2 * N + 1
    lab = [0 if s % 2 == 0 else (s + 1) // 2 for s in range(S)]
    p = np.exp(lp)
    a = np.zeros(S)
    a[0], a[1] = p[0, 0], p[0, lab[1]]
    for m in range(1, M):
        n = np.zeros(S)
        for s in range(S):
            v = a[s] + (a[s - 1] if s >= 1 else 0.0) + (a[s - 2] if s >= 3 and s % 2 == 1 else 0.0)
            n[s] = v * p[m, lab[s]]
        a = n
    return -np.log(a[S - 1] + a[S - 2])


def log_soft32(logp_row_block: np.ndarray) -> np.ndarray:
    """[M, N] float32 -> log softmax as the MAS kernel computes it: lse per row from the float64 exps of the float32
    differences, summed in phoneme order, rounded once; then a float32 subtraction."""
    x = np.asarray(logp_row_block, dtype=np.float32)
    m = x.max(axis=1)
    s = np.zeros(x.shape[0])
    for t in range(x.shape[1]):
        s += np.exp(x[:, t].astype(np.float64) - m.astype(np.float64))
    lse = (m.astype(np.float64) + np.log(s)).astype(np.float32)
    return x - lse[:, None]


def mas_width1(ls: np.ndarray) -> np.ndarray:
    """FastPitch's mas_width1 on log soft [M, N] float32 -> path [M] (phoneme of each frame): row 0 starts at t = 0,
    v[l, t] = ls[l, t] + max(v[l-1, t], v[l-1, t-1]) with the t - 1 predecessor winning ties, backtracked from
    (M - 1, N - 1).  Float32 throughout."""
    ls = np.asarray(ls, dtype=np.float32)
    M, N = ls.shape
    v = np.full(N, -np.inf, dtype=np.float32)
    v[0] = ls[0, 0]
    prev = np.zeros((M, N), dtype=np.int64)
    for i in range(1, M):
        left = np.concatenate([np.array([-np.inf], np.float32), v[:-1]])
        take = np.zeros(N, dtype=bool)
        take[1:] = left[1:] >= v[1:]
        prev[i] = np.arange(N) - take
        v = (ls[i] + np.where(take, left, v)).astype(np.float32)
    path = np.zeros(M, dtype=np.int64)
    j = N - 1
    for i in range(M - 1, -1, -1):
        path[i] = j
        j = prev[i, j]
    return path


def mas(logp32: np.ndarray, ilens, olens):
    """(durations [B, T] int64, path [B, L] int32 with -1 past olens) of float32 logp [B, L, T]."""
    B, L, T = logp32.shape
    dur = np.zeros((B, T), np.int64)
    path = np.full((B, L), -1, np.int32)
    for b in range(B):
        N, M = int(ilens[b]), int(olens[b])
        if M < N:
            continue
        p = mas_width1(log_soft32(logp32[b, :M, :N]))
        path[b, :M] = p
        dur[b] = np.bincount(p, minlength=T)
    return dur, path


def bin_loss(logp: torch.Tensor, path, ilens, olens) -> torch.Tensor:
    """[B] float64: -sum_l log(max(softmax_{t<N}(logp)[l, path[l]], 1e-12)) / M."""
    out = []
    for b in range(logp.shape[0]):
        N, M = int(ilens[b]), int(olens[b])
        soft = torch.softmax(logp[b, :M, :N], dim=1)
        idx = torch.as_tensor(np.asarray(path[b][:M]), dtype=torch.int64)
        out.append(-torch.log(torch.clamp(soft[torch.arange(M), idx], min=1e-12)).sum() / M)
    return torch.stack(out)


def loss(sd: dict, xs, ilens, mels, olens, bin_weight: float, path=None):
    """(total, forward-sum mean, bin mean) in float64 with gradients into a float64 copy of sd's parameters (returned as
    the fourth element, name -> leaf tensor).  path: the MAS path to use for the binarization loss (the kernel's, so both
    sides take the same path); None computes it from this model's own float32-rounded logp."""
    params = {n: v.detach().double().cpu().clone().requires_grad_(True) for n, v in sd.items()}
    k, q = keys_queries(params, xs, ilens, mels, olens)
    lp = logprob(q, k, ilens, olens)
    fs = forward_sum(lp, ilens, olens).mean()
    if path is None:
        path = mas(lp.detach().float().numpy(), ilens, olens)[1]
    bl = bin_loss(lp, path, ilens, olens).mean()
    total = fs + bin_weight * bl
    return total, fs, bl, params
