"""Float64 numpy restatement of the objective evaluation (DESIGN.md section 20): log-mel DCT cepstra, full DTW with its
path, MCD, and the prosody sums along the path, in the exact operation order the kernels use (every product and sum
rounded on its own, sums over increasing m / k), so cepstra, costs, paths and MCD match the GPU bit for bit.

The DTW is vectorised over anti-diagonals: every cell of a diagonal depends only on the two diagonals before it."""
from __future__ import annotations

import math

import numpy as np

MCD_SCALE = 10.0 * math.sqrt(2.0) / math.log(10.0)
DIAG, UP, LEFT = 0, 1, 2          # predecessor (i-1, j-1), (i-1, j), (i, j-1)


def cepstra(mel: np.ndarray, D: np.ndarray) -> np.ndarray:
    """mel [T, M] (any float), D [M, K] float64 -> c [T, K] = sum over increasing m of double(mel[:, m]) * D[m]."""
    mel = np.asarray(mel, dtype=np.float64)
    acc = np.zeros((mel.shape[0], D.shape[1]), dtype=np.float64)
    for m in range(D.shape[0]):
        acc = acc + mel[:, m:m + 1] * D[m][None, :]
    return acc


def distances(cx: np.ndarray, cy: np.ndarray, i: np.ndarray, j: np.ndarray) -> np.ndarray:
    """d(i, j) = sqrt(sum over increasing k of (cx[i, k] - cy[j, k])^2) for index arrays i, j."""
    acc = np.zeros(len(i), dtype=np.float64)
    for k in range(cx.shape[1]):
        diff = cx[i, k] - cy[j, k]
        acc = acc + diff * diff
    return np.sqrt(acc)


def dtw(cx: np.ndarray, cy: np.ndarray):
    """cx [Lx, K], cy [Ly, K] float64 -> (cost A(Lx-1, Ly-1), path [P, 2] int64 from (0, 0), A [Lx, Ly])."""
    Lx, Ly = cx.shape[0], cy.shape[0]
    A = np.full((Lx, Ly), np.nan)
    direction = np.zeros((Lx, Ly), dtype=np.int8)
    for s in range(Lx + Ly - 1):
        i = np.arange(max(0, s - (Ly - 1)), min(s, Lx - 1) + 1)
        j = s - i
        d = distances(cx, cy, i, j)
        best = np.zeros(len(i))
        dv = np.full(len(i), DIAG, dtype=np.int8)
        have = (i > 0) & (j > 0)
        best[have] = A[i[have] - 1, j[have] - 1]
        for cand, (di, dj), code in ((i > 0, (1, 0), UP), (j > 0, (0, 1), LEFT)):
            v = np.zeros(len(i))
            v[cand] = A[i[cand] - di, j[cand] - dj]
            take = cand & (~have | (v < best))
            best[take], dv[take] = v[take], code
            have = have | cand
        A[i, j] = np.where(have, d + best, d)
        direction[i, j] = dv
    path = [(Lx - 1, Ly - 1)]
    i, j = Lx - 1, Ly - 1
    while i + j > 0:
        dv = direction[i, j]
        i, j = i - (dv != LEFT), j - (dv != UP)
        path.append((i, j))
    return A[Lx - 1, Ly - 1], np.array(path[::-1], dtype=np.int64), A


def mcd(cost: float, P: int, scale: float = MCD_SCALE) -> float:
    return (np.float64(cost) / np.float64(P)) * np.float64(scale)


def prosody(path: np.ndarray, f0x: np.ndarray, f0y: np.ndarray, ex: np.ndarray, ey: np.ndarray):
    """Walk path [P, 2] in order; f0x / f0y are the F0 contours up to their own lengths (cells past them are unvoiced).
    -> (counts (P, n_vuv, n_voiced, n_gross), sums (sq_cents, sq_energy))."""
    n_vuv = n_voiced = n_gross = 0
    sq_cents = sq_energy = np.float64(0.0)
    for i, j in path:
        fx = np.float64(f0x[i]) if i < len(f0x) else np.float64(0.0)
        fy = np.float64(f0y[j]) if j < len(f0y) else np.float64(0.0)
        vx, vy = fx > 0, fy > 0
        n_vuv += int(vx != vy)
        if vx and vy:
            n_voiced += 1
            r = fx / fy
            c = np.float64(1200.0) * np.log2(r)
            sq_cents = sq_cents + c * c
            n_gross += int(abs(r - 1.0) > 0.2)
        e = np.float64(ex[i]) - np.float64(ey[j])
        sq_energy = sq_energy + e * e
    return (len(path), n_vuv, n_voiced, n_gross), (float(sq_cents), float(sq_energy))


def evaluate_pair(xmel: np.ndarray, ymel: np.ndarray, D: np.ndarray, f0x=None, f0y=None, ex=None, ey=None,
                  scale: float = MCD_SCALE) -> dict:
    """One pair, [T, M] log-mels each -> {"mcd", "cost", "plen", "path"[, "counts", "sums"]}."""
    cost, path, _ = dtw(cepstra(xmel, D), cepstra(ymel, D))
    out = {"mcd": float(mcd(cost, len(path), scale)), "cost": float(cost), "plen": len(path), "path": path}
    if f0x is not None:
        out["counts"], out["sums"] = prosody(path, f0x, f0y, ex, ey)
    return out


def backend(n_cep: int, log=None):
    """The evaluate command's device entry restated on this oracle: score(pairs, with_prosody) -> per-utterance rows.
    `log`, when given, collects each batch's ids."""
    from fastspeech2_b200.evaluate import COUNT_FIELDS, SUM_FIELDS, dct_basis

    def score(bt, with_prosody):
        if log is not None:
            log.append([u["id"] for u in bt])
        rows = []
        for u in bt:
            r = evaluate_pair(u["x"], u["y"], dct_basis(u["x"].shape[1], n_cep), u["f0x"], u["f0y"], u["ex"], u["ey"])
            rows.append({"mcd_db": r["mcd"], "cost": r["cost"], **dict(zip(COUNT_FIELDS, r["counts"])),
                         **dict(zip(SUM_FIELDS, r["sums"]))})
        return rows
    return score
