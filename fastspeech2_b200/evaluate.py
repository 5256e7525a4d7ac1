"""Objective evaluation on the GPU (DESIGN.md section 20): mel-cepstral distortion under a full DTW alignment, and F0,
voicing and energy errors along the alignment path, for a ragged batch of (synthesized, reference) pairs.

    python -m fastspeech2_b200.evaluate --ref DATA_DIR --syn SYN_DIR [--ids FILE] [--n-cep 24] [--csv OUT] [--budget CELLS]

The directories are what `python -m fastspeech2_b200.preprocess` writes: mels/{id}.npy [n_mels, T] float32, and, where
both sides have them, pitch/{id}.npy float64 and energy/{id}.npy float32.  It prints one JSON line of dataset figures:

  mcd_db         mean over utterances of MCD_b = A(Lx-1, Ly-1) / P * 10 sqrt(2) / ln 10
  f0_rmse_cents  sqrt(sum sq_cents / sum n_voiced)        gpe  sum n_gross / sum n_voiced
  vuv_error      sum n_vuv / sum P                        ffe  (sum n_vuv + sum n_gross) / sum P
  energy_rmse    sqrt(sum sq_energy / sum P)              length_ratio  mean over utterances of Lx / Ly

The cepstra are c1..c_{n_cep} of the orthonormal DCT-II of each log-mel frame (c0, the frame's level, dropped): these
numbers are not comparable with MCD computed on WORLD / SPTK mel-cepstra.  Cepstra, DTW costs, paths and MCD are
bit-identical to a float64 restatement (oracle/eval_oracle.py); each pair's results do not depend on its batch mates."""
from __future__ import annotations

import argparse
import csv
import json
import math
import os
import queue
import threading

import numpy as np
import torch

from . import _lib
from ._kernel_module import check_status, query_bytes, workspace

MCD_SCALE = 10.0 * math.sqrt(2.0) / math.log(10.0)
N_CEP = 24
COUNT_FIELDS = ("path_len", "n_vuv", "n_voiced", "n_gross")
SUM_FIELDS = ("sq_cents", "sq_energy")

_ws: dict = {}        # device index -> workspace tensor
_dct: dict = {}       # (n_mels, n_cep, device index) -> the basis on that device


def dct_basis(n_mels: int, n_cep: int) -> np.ndarray:
    """D [n_mels, n_cep] float64, D[m, k-1] = sqrt(2/M) cos(pi k (m + 1/2) / M) for k = 1..n_cep: the orthonormal DCT-II
    without c0."""
    m = np.arange(n_mels, dtype=np.float64)[:, None]
    k = np.arange(1, n_cep + 1, dtype=np.float64)[None, :]
    return np.sqrt(2.0 / n_mels) * np.cos(np.pi * k * (m + 0.5) / n_mels)


def workspace_bytes(B: int, Lx_max: int, Ly_max: int, n_mels: int = 80, n_cep: int = N_CEP, with_path: bool = False) -> int:
    """Bytes of device workspace an mcd_dtw call needs; without a path it grows with Lx_max + Ly_max, not their product."""
    return query_bytes("fs2_dtw_workspace_bytes", int(B), int(Lx_max), int(Ly_max), int(n_mels), int(n_cep), int(bool(with_path)))


def _is_int(t) -> bool:
    return not (t.dtype.is_floating_point or t.dtype.is_complex or t.dtype == torch.bool)


def _lens(name: str, t, B: int) -> None:
    if not torch.is_tensor(t) or t.dim() != 1 or t.shape[0] != B:
        raise ValueError(f"{name} must be a [B={B}] tensor")
    if not _is_int(t):
        raise ValueError(f"{name} must be an integer tensor (got {t.dtype})")


def _check_cuda(names: str, *ts) -> torch.device:
    dev = ts[0].device
    if not all(t.is_cuda and t.device == dev for t in ts):
        raise ValueError(f"{names} must be CUDA tensors on one device (the H100 path has no CPU fallback)")
    return dev


def _check_mcd_args(x, xlens, y, ylens, n_cep):
    for name, t in (("x", x), ("y", y)):
        if not torch.is_tensor(t) or t.dim() != 3 or min(t.shape) == 0:
            raise ValueError(f"{name} must be a non-empty [B, L, n_mels] tensor")
        if t.dtype != torch.float32:
            raise ValueError(f"{name} must be float32 log-mels (got {t.dtype})")
    B, _, M = x.shape
    if y.shape[0] != B:
        raise ValueError(f"y has {y.shape[0]} utterances, x has {B}")
    if y.shape[2] != M:
        raise ValueError(f"y has n_mels={y.shape[2]}, x has n_mels={M}")
    _lens("xlens", xlens, B)
    _lens("ylens", ylens, B)
    if isinstance(n_cep, bool) or not isinstance(n_cep, (int, np.integer)) or not 1 <= n_cep <= M - 1:
        raise ValueError(f"n_cep must be an integer in [1, n_mels - 1 = {M - 1}] (got {n_cep!r})")
    return B, M


def mcd_dtw(x: torch.Tensor, xlens: torch.Tensor, y: torch.Tensor, ylens: torch.Tensor, *, n_cep: int = N_CEP,
            return_path: bool = False):
    """x [B, Lx_max, M] synthesized and y [B, Ly_max, M] reference log-mels (fp32, CUDA) with their frame counts ->
    (mcd [B] float64 dB, cost [B] float64, plen [B] int64[, path [B, Lx_max + Ly_max - 1, 2] int32, -1 past plen]).
    Rows at or past a length are never read."""
    B, M = _check_mcd_args(x, xlens, y, ylens, n_cep)
    dev = _check_cuda("x, xlens, y and ylens", x, xlens, y, ylens)
    x, y = x.contiguous(), y.contiguous()
    xlens, ylens = xlens.to(torch.int64).contiguous(), ylens.to(torch.int64).contiguous()
    Lx, Ly = x.shape[1], y.shape[1]
    key = (M, int(n_cep), dev.index)
    if key not in _dct:
        _dct[key] = torch.from_numpy(dct_basis(M, int(n_cep))).to(dev)
    ws = workspace(_ws, dev, workspace_bytes(B, Lx, Ly, M, n_cep, return_path))
    mcd = torch.empty(B, dtype=torch.float64, device=dev)
    cost = torch.empty(B, dtype=torch.float64, device=dev)
    plen = torch.empty(B, dtype=torch.int64, device=dev)
    path = torch.empty((B, Lx + Ly - 1, 2), dtype=torch.int32, device=dev) if return_path else None
    status = torch.empty((1,), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().fs2_mcd_dtw(_lib.ptr(x), _lib.ptr(xlens), Lx, _lib.ptr(y), _lib.ptr(ylens), Ly, B, M,
                                           _lib.ptr(_dct[key]), int(n_cep), MCD_SCALE, _lib.ptr(mcd), _lib.ptr(cost),
                                           _lib.ptr(plen), _lib.ptr(path), _lib.ptr(status), _lib.ptr(ws), ws.numel(),
                                           _lib.stream_ptr(dev)), "fs2_mcd_dtw")
    check_status(status, [
        (_lib.FS2_EVAL_BAD_LENGTH, f"every xlens[b] must lie in [1, Lx_max={Lx}] and every ylens[b] in [1, Ly_max={Ly}]"),
        (_lib.FS2_EVAL_NONFINITE, "x and y must be finite log-mels within their lengths (found NaN or inf)")])
    return (mcd, cost, plen, path) if return_path else (mcd, cost, plen)


def path_prosody(path, plen, f0x, f0x_lens, f0y, f0y_lens, ex, ey):
    """Walk each path[b, :plen[b]] (as mcd_dtw returns it) in order, with F0 contours f0x [B, Fx] / f0y [B, Fy] float64 up
    to their lengths (frames past them are unvoiced) and energies ex [B, Ex] / ey [B, Ey] float32 ->
    (counts [B, 4] int64: P, n_vuv, n_voiced, n_gross;  sums [B, 2] float64: sq_cents, sq_energy)."""
    if not torch.is_tensor(path) or path.dim() != 3 or path.shape[2] != 2 or min(path.shape) == 0:
        raise ValueError("path must be a non-empty [B, P_max, 2] tensor")
    if path.dtype != torch.int32:
        raise ValueError(f"path must be int32 (got {path.dtype})")
    B = path.shape[0]
    _lens("plen", plen, B)
    for name, t, dt in (("f0x", f0x, torch.float64), ("f0y", f0y, torch.float64), ("ex", ex, torch.float32), ("ey", ey, torch.float32)):
        if not torch.is_tensor(t) or t.dim() != 2 or t.shape[0] != B or t.shape[1] == 0:
            raise ValueError(f"{name} must be a non-empty [B={B}, L] tensor")
        if t.dtype != dt:
            raise ValueError(f"{name} must be {dt} (got {t.dtype})")
    _lens("f0x_lens", f0x_lens, B)
    _lens("f0y_lens", f0y_lens, B)
    dev = _check_cuda("path, plen, f0x, f0x_lens, f0y, f0y_lens, ex and ey", path, plen, f0x, f0x_lens, f0y, f0y_lens, ex, ey)
    path, f0x, f0y, ex, ey = (t.contiguous() for t in (path, f0x, f0y, ex, ey))
    plen, f0x_lens, f0y_lens = (t.to(torch.int64).contiguous() for t in (plen, f0x_lens, f0y_lens))
    counts = torch.empty((B, 4), dtype=torch.int64, device=dev)
    sums = torch.empty((B, 2), dtype=torch.float64, device=dev)
    status = torch.empty((1,), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().fs2_path_prosody(_lib.ptr(path), _lib.ptr(plen), B, path.shape[1], _lib.ptr(f0x), _lib.ptr(f0x_lens),
                                                f0x.shape[1], _lib.ptr(f0y), _lib.ptr(f0y_lens), f0y.shape[1], _lib.ptr(ex),
                                                ex.shape[1], _lib.ptr(ey), ey.shape[1], _lib.ptr(counts), _lib.ptr(sums),
                                                _lib.ptr(status), _lib.stream_ptr(dev)), "fs2_path_prosody")
    check_status(status, [(_lib.FS2_EVAL_BAD_LENGTH, "plen must lie in [0, P_max], F0 lengths within f0x / f0y, and path cells "
                                                     "within ex / ey")])
    return counts, sums


# ---- dataset figures ------------------------------------------------------------------------------------------------

def _ratio(num, den):
    return float(num) / float(den) if den else None


def dataset_figures(rows, pitch: bool = True, energy: bool = True) -> dict:
    """Per-utterance rows (dicts with lx, ly, mcd_db and the COUNT_FIELDS / SUM_FIELDS) -> the command's figures; the F0
    figures are None without pitch on both sides, energy_rmse without energy, and a ratio with a zero denominator."""
    out = {"utterances": len(rows),
           "mcd_db": float(np.mean([r["mcd_db"] for r in rows])) if rows else None,
           "length_ratio": float(np.mean([r["lx"] / r["ly"] for r in rows])) if rows else None}
    P = sum(r["path_len"] for r in rows)
    vuv, voiced, gross = (sum(r[k] for r in rows) for k in ("n_vuv", "n_voiced", "n_gross"))
    sq_cents = math.fsum(r["sq_cents"] for r in rows)
    sq_energy = math.fsum(r["sq_energy"] for r in rows)
    f0 = pitch and bool(rows)
    out["f0_rmse_cents"] = math.sqrt(sq_cents / voiced) if f0 and voiced else None
    out["vuv_error"] = _ratio(vuv, P) if f0 else None
    out["gpe"] = _ratio(gross, voiced) if f0 else None
    out["ffe"] = _ratio(vuv + gross, P) if f0 else None
    out["energy_rmse"] = math.sqrt(sq_energy / P) if energy and P else None
    return out


# ---- the command ----------------------------------------------------------------------------------------------------

def _load(path: str) -> np.ndarray:
    if not os.path.exists(path):
        raise FileNotFoundError(f"missing file {path}")
    return np.load(path, allow_pickle=False)


def read_pair(ref_dir: str, syn_dir: str, uid: str, pitch: bool, energy: bool) -> dict:
    """One utterance's arrays: x / y [T, n_mels] float32 (the files are [n_mels, T]), and f0 / energy where asked."""
    u = {"id": uid, "x": np.ascontiguousarray(_load(os.path.join(syn_dir, "mels", uid + ".npy")).T, dtype=np.float32),
         "y": np.ascontiguousarray(_load(os.path.join(ref_dir, "mels", uid + ".npy")).T, dtype=np.float32)}
    for side, d in (("x", syn_dir), ("y", ref_dir)):
        T = u[side].shape[0]
        u["f0" + side] = _load(os.path.join(d, "pitch", uid + ".npy")).astype(np.float64) if pitch else np.zeros(0)
        if energy:
            e = _load(os.path.join(d, "energy", uid + ".npy")).astype(np.float32)
            if e.shape != (T,):
                raise ValueError(f"{os.path.join(d, 'energy', uid + '.npy')}: {e.shape[0]} frames, its mel has {T}")
            u["e" + side] = e
        else:
            u["e" + side] = np.zeros(T, dtype=np.float32)
    return u


def batches(pairs, budget: int):
    """Yield lists of pairs whose padded DTW grid B * Lx_max * Ly_max stays within `budget` cells (a larger pair goes
    alone)."""
    cur, lx, ly = [], 0, 0
    for u in pairs:
        mx, my = max(lx, u["x"].shape[0]), max(ly, u["y"].shape[0])
        if cur and (len(cur) + 1) * mx * my > budget:
            yield cur
            cur, mx, my = [], u["x"].shape[0], u["y"].shape[0]
        cur.append(u)
        lx, ly = mx, my
    if cur:
        yield cur


def gpu_backend(n_cep: int = N_CEP, device="cuda"):
    """score(list of pairs, with_prosody) -> list of per-utterance rows on the library's kernels."""

    def pad(arrs, dtype, tail=()):
        n = [a.shape[0] for a in arrs]
        out = np.zeros((len(arrs), max(max(n), 1)) + tail, dtype=dtype)
        for b, a in enumerate(arrs):
            out[b, : n[b]] = a
        return torch.from_numpy(out).to(device), torch.tensor(n, dtype=torch.int64, device=device)

    def score(bt, with_prosody: bool):
        M = bt[0]["x"].shape[1]
        x, xl = pad([u["x"] for u in bt], np.float32, (M,))
        y, yl = pad([u["y"] for u in bt], np.float32, (M,))
        res = mcd_dtw(x, xl, y, yl, n_cep=n_cep, return_path=with_prosody)
        if with_prosody:
            fx, fxl = pad([u["f0x"] for u in bt], np.float64)
            fy, fyl = pad([u["f0y"] for u in bt], np.float64)
            ex, _ = pad([u["ex"] for u in bt], np.float32)
            ey, _ = pad([u["ey"] for u in bt], np.float32)
            counts, sums = (t.cpu().numpy() for t in path_prosody(res[3], res[2], fx, fxl, fy, fyl, ex, ey))
        else:
            counts, sums = np.zeros((len(bt), 4), dtype=np.int64), np.zeros((len(bt), 2))
            counts[:, 0] = res[2].cpu().numpy()
        mcd, cost = res[0].cpu().numpy(), res[1].cpu().numpy()
        return [{"mcd_db": float(mcd[b]), "cost": float(cost[b]), **dict(zip(COUNT_FIELDS, map(int, counts[b]))),
                 **dict(zip(SUM_FIELDS, map(float, sums[b])))} for b in range(len(bt))]
    return score


def list_ids(syn_dir: str, ids_file: str = None) -> list:
    """The ids of --ids (one per line, up to a '|'; blank lines skipped), else every mels/*.npy of syn_dir, sorted."""
    if ids_file:
        with open(ids_file) as f:
            return [ln.split("|")[0].strip() for ln in f if ln.split("|")[0].strip()]
    d = os.path.join(syn_dir, "mels")
    if not os.path.isdir(d):
        raise FileNotFoundError(f"missing directory {d}")
    return sorted(n[:-4] for n in os.listdir(d) if n.endswith(".npy"))


def run(ref_dir: str, syn_dir: str, ids=None, n_cep: int = N_CEP, csv_path: str = None, budget: int = 1 << 28,
        score=None) -> dict:
    """Score syn_dir against ref_dir; returns the dataset figures.  `score` replaces the GPU backend (a function from a
    list of pairs and a with-prosody flag to a list of per-utterance rows)."""
    ids = list_ids(syn_dir) if ids is None else list(ids)
    has = lambda k: all(os.path.isdir(os.path.join(d, k)) for d in (ref_dir, syn_dir))   # noqa: E731
    pitch, energy = has("pitch"), has("energy")
    score = score or gpu_backend(n_cep)
    q: queue.Queue = queue.Queue(maxsize=2)       # a reader thread keeps one batch ahead of the GPU

    def reader():
        try:
            for bt in batches((read_pair(ref_dir, syn_dir, u, pitch, energy) for u in ids), budget):
                q.put(bt)
            q.put(None)
        except BaseException as e:                # re-raised in the consumer
            q.put(e)
    th = threading.Thread(target=reader, daemon=True)
    th.start()
    rows = []
    while True:
        bt = q.get()
        if bt is None:
            break
        if isinstance(bt, BaseException):
            raise bt
        for u, r in zip(bt, score(bt, pitch or energy)):
            rows.append({"id": u["id"], "lx": u["x"].shape[0], "ly": u["y"].shape[0], **r})
    th.join()
    if csv_path:
        with open(csv_path, "w", newline="") as f:
            w = csv.DictWriter(f, fieldnames=["id", "lx", "ly", "mcd_db", "cost", *COUNT_FIELDS, *SUM_FIELDS])
            w.writeheader()
            for r in rows:
                w.writerow(r)
    out = dataset_figures(rows, pitch, energy)
    out["n_cep"] = int(n_cep)
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--ref", required=True, help="reference features (preprocess output: mels/, pitch/, energy/)")
    ap.add_argument("--syn", required=True, help="features of the synthesized wavs, same layout")
    ap.add_argument("--ids", default=None, help="file of utterance ids, one per line (default: every SYN/mels/*.npy)")
    ap.add_argument("--n-cep", type=int, default=N_CEP, help="cepstra c1..c_n compared (default 24)")
    ap.add_argument("--csv", default=None, help="write one row per utterance here")
    ap.add_argument("--budget", type=int, default=1 << 28, help="DTW cells per GPU batch, padding included")
    args = ap.parse_args(argv)
    ids = list_ids(args.syn, args.ids)
    print(json.dumps(run(args.ref, args.syn, ids, args.n_cep, args.csv, args.budget)))


if __name__ == "__main__":
    main()
