"""Phoneme durations without an external aligner (DESIGN.md section 24): the unsupervised alignment module of Badlani et
al., "One TTS Alignment To Rule Them All" (2021), as FastPitch 1.1 builds it, trained and run on the library's kernels.

    python -m fastspeech2_b200.aligner train   -c config.yaml --filelist FILE [-d DATA_DIR] [--steps N] [--batch B] [--bin-start S] -o aligner.pt
    python -m fastspeech2_b200.aligner extract -c config.yaml --filelist FILE [-d DATA_DIR] -p aligner.pt --out NEW_FILELIST

Filelist lines are the reference's five `|` fields: text, boundaries, durations, phonemes, wav name (fields 1 and 2 may
be empty), optionally followed by a sixth, the speaker name (`python -m fastspeech2_b200.speakers tag`), which `extract`
carries through.  Mels are read from `{data_dir}/mels/{id}.npy` of a `preprocess` tree, id = the wav name up to its first dot,
as the reference's `TTSDataset` does.  `extract` writes the same lines with field 2 replaced by the durations found by
monotonic alignment search, which sum to the mel's frame count, so the reference's loader trains on them unchanged (its
last-duration correction then changes nothing).  Field 1 becomes the start frame 0 followed by the cumulative end frame
of every phoneme, the layout of the reference's LJSpeech lines; the reference's loader does not read it.  Lines with more
phonemes than frames are reported and skipped.  When the input lines carry durations, `extract` also prints one JSON
line of agreement with them.

`Aligner(n_symbols)` holds parameters only.  Text side: Embedding(n, 256, padding 0), Conv1d(256, 512, 3) + ReLU,
Conv1d(512, 80, 1) -> keys k [B, T, 80].  Mel side, on the log-mels as `preprocess` writes them: Conv1d(80, 160, 3) +
ReLU, Conv1d(160, 80, 1) + ReLU, Conv1d(80, 80, 1) -> queries q [B, L, 80].  Rows at or past an utterance's length are
zeroed before every convolution, so an utterance's result does not depend on its batch mates.  The convolutions run on
`train.ConvFn` in TF32, the embedding on `train.EmbedFn`; the attention, losses and MAS on csrc/aligner.cu."""
from __future__ import annotations

import argparse
import json
import os
import sys
from typing import List, Optional, Sequence

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from . import train as _train
from ._kernel_module import query_bytes, workspace
from .data import BucketBatchSampler
from .optim import NoamAdam

EMB, HID, ATT, N_MELS = 256, 512, _lib.FS2_ALIGN_DIM, 80
STATUS_MESSAGES = [(_lib.FS2_ALIGN_BAD_LENGTH, "lengths outside [1, T] / [1, L] (or a path index outside the phonemes)"),
                   (_lib.FS2_ALIGN_INFEASIBLE, "more phonemes than frames"),
                   (_lib.FS2_ALIGN_NONFINITE, "NaN or inf in the inputs")]


# ---- filelists -------------------------------------------------------------------------------------------------------
class Line:
    """One filelist line: text | boundaries | durations | phonemes | wav name [| speaker name]."""
    __slots__ = ("text", "boundaries", "durations", "phonemes", "wav", "speaker")

    def __init__(self, text: str, boundaries: Optional[List[int]], durations: Optional[List[int]], phonemes: List[str], wav: str,
                 speaker: Optional[str] = None):
        self.text, self.boundaries, self.durations, self.phonemes, self.wav = text, boundaries, durations, phonemes, wav
        self.speaker = speaker

    @property
    def id(self) -> str:
        return self.wav.split(".")[0]


def parse_line(line: str, where: str = "line") -> Line:
    """A filelist line -> Line; empty fields 1 and 2 give None, and a line without the sixth (speaker) field gives
    speaker None.  Raises ValueError naming `where` on a malformed line."""
    f = line.rstrip("\r\n").split("|")
    if len(f) not in (5, 6):
        raise ValueError(f"{where}: expected 5 '|'-separated fields, found {len(f)} (a sixth, the speaker name, is optional)")
    speaker = None
    if len(f) == 6:
        speaker = f[5].strip()
        if not speaker:
            raise ValueError(f"{where}: empty speaker field")
    ints = []
    for k in (1, 2):
        try:
            ints.append([int(v) for v in f[k].split()] or None)
        except ValueError:
            raise ValueError(f"{where}: field {k + 1} must hold integers") from None
    phonemes = f[3].split()
    if not phonemes:
        raise ValueError(f"{where}: no phonemes")
    if not f[4].strip():
        raise ValueError(f"{where}: no wav name")
    if ints[1] is not None and len(ints[1]) != len(phonemes):
        raise ValueError(f"{where}: {len(ints[1])} durations for {len(phonemes)} phonemes")
    return Line(f[0], ints[0], ints[1], phonemes, f[4].strip(), speaker)


def read_filelist(path: str) -> List[Line]:
    with open(path, encoding="utf-8") as fh:
        return [parse_line(ln, f"{path}:{i + 1}") for i, ln in enumerate(fh) if ln.strip()]


def format_line(line: Line, durations: Sequence[int]) -> str:
    """`line` with field 2 = durations and field 1 = 0 followed by their cumulative end frames (and its speaker field,
    if it has one)."""
    d = [int(v) for v in durations]
    ends = np.cumsum([0] + d).tolist()
    fields = [line.text, " ".join(map(str, ends)), " ".join(map(str, d)), " ".join(line.phonemes), line.wav]
    return "|".join(fields + ([line.speaker] if line.speaker is not None else []))


def build_symbols(lines: Sequence[Line]) -> List[str]:
    """The symbol table: "<pad>" (id 0) then the sorted set of phoneme tokens in `lines`."""
    return ["<pad>"] + sorted({p for ln in lines for p in ln.phonemes})


def encode(line: Line, symbols: Sequence[str]) -> np.ndarray:
    table = {s: i for i, s in enumerate(symbols)}
    missing = sorted({p for p in line.phonemes if p not in table or p == "<pad>"})
    if missing:
        raise ValueError(f"{line.wav}: phonemes {missing} are not in the aligner's symbol table")
    return np.array([table[p] for p in line.phonemes], dtype=np.int64)


def load_mel(data_dir: str, line: Line) -> np.ndarray:
    """[L, 80] float32 from {data_dir}/mels/{id}.npy ([80, L] as preprocess writes it)."""
    m = np.load(os.path.join(data_dir, "mels", line.id + ".npy"))
    if m.ndim != 2 or m.shape[0] != N_MELS:
        raise ValueError(f"{line.id}: mel has shape {m.shape}, expected [{N_MELS}, frames]")
    return np.ascontiguousarray(m.T, dtype=np.float32)


# ---- autograd functions over csrc/aligner.cu -------------------------------------------------------------------------
def workspace_bytes(B: int, L: int, T: int) -> int:
    """Bytes of the workspace every fs2_align_* entry takes for a [B, L, T] call."""
    return query_bytes("fs2_align_workspace_bytes", int(B), int(L), int(T))


_WS: dict = {}


def _ws(device, B, L, T) -> torch.Tensor:
    return workspace(_WS, device, workspace_bytes(B, L, T))


def _slot(status: torch.Tensor, i: int) -> int:
    return status.data_ptr() + 4 * i


class MaskRowsFn(torch.autograd.Function):
    """x [B, L, C] with rows t >= lens[b] set to +0; the gradient is masked the same way."""

    @staticmethod
    def forward(ctx, x, lens):
        x = _train._c(x)
        B, L, C = x.shape
        y = torch.empty_like(x)
        _lib.check(_lib.load().fs2_align_mask_rows(x.data_ptr(), lens.data_ptr(), B, L, C, y.data_ptr(), _train._st(x)), "fs2_align_mask_rows")
        ctx.save_for_backward(lens)
        return y

    @staticmethod
    def backward(ctx, dy):
        (lens,) = ctx.saved_tensors
        dy = _train._c(dy)
        B, L, C = dy.shape
        dx = torch.empty_like(dy)
        _lib.check(_lib.load().fs2_align_mask_rows(dy.data_ptr(), lens.data_ptr(), B, L, C, dx.data_ptr(), _train._st(dy)), "fs2_align_mask_rows")
        return dx, None


class AlignLogProbFn(torch.autograd.Function):
    """logp [B, L, T] from q [B, L, 80], k [B, T, 80] (fs2_align_logprob); backward fs2_align_logprob_backward.
    status: int32 device tensor, slots 0 (forward) and 1 (backward) are written."""

    @staticmethod
    def forward(ctx, q, k, ilens, olens, status):
        q, k = _train._c(q), _train._c(k)
        B, L, T = q.shape[0], q.shape[1], k.shape[1]
        ws = _ws(q.device, B, L, T)
        logp = torch.empty((B, L, T), dtype=torch.float32, device=q.device)
        _lib.check(_lib.load().fs2_align_logprob(q.data_ptr(), k.data_ptr(), ilens.data_ptr(), olens.data_ptr(), B, L, T, logp.data_ptr(),
                                                 _slot(status, 0), ws.data_ptr(), ws.numel(), _train._st(q)), "fs2_align_logprob")
        ctx.save_for_backward(q, k, ilens, olens, status)
        return logp

    @staticmethod
    def backward(ctx, dlogp):
        q, k, ilens, olens, status = ctx.saved_tensors
        dlogp = _train._c(dlogp)
        B, L, T = dlogp.shape
        ws = _ws(q.device, B, L, T)
        dq, dk = torch.empty_like(q), torch.empty_like(k)
        _lib.check(_lib.load().fs2_align_logprob_backward(q.data_ptr(), k.data_ptr(), ilens.data_ptr(), olens.data_ptr(), B, L, T,
                                                          dlogp.data_ptr(), dq.data_ptr(), dk.data_ptr(), _slot(status, 1), ws.data_ptr(),
                                                          ws.numel(), _train._st(q)), "fs2_align_logprob_backward")
        return dq, dk, None, None, None


class ForwardSumFn(torch.autograd.Function):
    """Per-utterance forward-sum loss [B] (fs2_align_forward_sum); the backward reruns the lattice with the incoming
    gradient as dloss and writes dlogp.  Status slots 2 and 3."""

    @staticmethod
    def forward(ctx, logp, ilens, olens, status):
        logp = _train._c(logp)
        B, L, T = logp.shape
        ws = _ws(logp.device, B, L, T)
        loss = torch.empty((B,), dtype=torch.float32, device=logp.device)
        _lib.check(_lib.load().fs2_align_forward_sum(logp.data_ptr(), ilens.data_ptr(), olens.data_ptr(), B, L, T, None, loss.data_ptr(), None,
                                                     _slot(status, 2), ws.data_ptr(), ws.numel(), _train._st(logp)), "fs2_align_forward_sum")
        ctx.save_for_backward(logp, ilens, olens, status)
        return loss

    @staticmethod
    def backward(ctx, g):
        logp, ilens, olens, status = ctx.saved_tensors
        g = _train._c(g)
        B, L, T = logp.shape
        ws = _ws(logp.device, B, L, T)
        loss = torch.empty((B,), dtype=torch.float32, device=logp.device)
        dlogp = torch.empty_like(logp)
        _lib.check(_lib.load().fs2_align_forward_sum(logp.data_ptr(), ilens.data_ptr(), olens.data_ptr(), B, L, T, g.data_ptr(), loss.data_ptr(),
                                                     dlogp.data_ptr(), _slot(status, 3), ws.data_ptr(), ws.numel(), _train._st(logp)),
                   "fs2_align_forward_sum")
        return dlogp, None, None, None


class BinLossFn(torch.autograd.Function):
    """Per-utterance binarization loss [B] on the MAS path (fs2_align_bin_loss).  Status slots 5 and 6."""

    @staticmethod
    def forward(ctx, logp, path, ilens, olens, status):
        logp = _train._c(logp)
        B, L, T = logp.shape
        ws = _ws(logp.device, B, L, T)
        loss = torch.empty((B,), dtype=torch.float32, device=logp.device)
        _lib.check(_lib.load().fs2_align_bin_loss(logp.data_ptr(), path.data_ptr(), ilens.data_ptr(), olens.data_ptr(), B, L, T, None,
                                                  loss.data_ptr(), None, _slot(status, 5), ws.data_ptr(), ws.numel(), _train._st(logp)),
                   "fs2_align_bin_loss")
        ctx.save_for_backward(logp, path, ilens, olens, status)
        return loss

    @staticmethod
    def backward(ctx, g):
        logp, path, ilens, olens, status = ctx.saved_tensors
        g = _train._c(g)
        B, L, T = logp.shape
        ws = _ws(logp.device, B, L, T)
        loss = torch.empty((B,), dtype=torch.float32, device=logp.device)
        dlogp = torch.empty_like(logp)
        _lib.check(_lib.load().fs2_align_bin_loss(logp.data_ptr(), path.data_ptr(), ilens.data_ptr(), olens.data_ptr(), B, L, T, g.data_ptr(),
                                                  loss.data_ptr(), dlogp.data_ptr(), _slot(status, 6), ws.data_ptr(), ws.numel(),
                                                  _train._st(logp)), "fs2_align_bin_loss")
        return dlogp, None, None, None, None


def mas(logp: torch.Tensor, ilens: torch.Tensor, olens: torch.Tensor, status: torch.Tensor, slot: int = 4):
    """(durations [B, T] int64, path [B, L] int32) of logp [B, L, T] (fs2_align_mas)."""
    logp = _train._c(logp)
    B, L, T = logp.shape
    ws = _ws(logp.device, B, L, T)
    dur = torch.empty((B, T), dtype=torch.int64, device=logp.device)
    path = torch.empty((B, L), dtype=torch.int32, device=logp.device)
    _lib.check(_lib.load().fs2_align_mas(logp.data_ptr(), ilens.data_ptr(), olens.data_ptr(), B, L, T, dur.data_ptr(), path.data_ptr(),
                                         _slot(status, slot), ws.data_ptr(), ws.numel(), _train._st(logp)), "fs2_align_mas")
    return dur, path


def status_bits(status: torch.Tensor) -> int:
    """OR of a status tensor's slots (one host read)."""
    return int(np.bitwise_or.reduce(status.cpu().numpy()))


def describe_status(bits: int) -> str:
    return "; ".join(msg for bit, msg in STATUS_MESSAGES if bits & bit)


# ---- the model -------------------------------------------------------------------------------------------------------
class Aligner(nn.Module):
    """The alignment module's parameters (module docstring); the computation runs in `keys_queries`, `loss` and
    `durations` on CUDA tensors only."""

    def __init__(self, n_symbols: int):
        super().__init__()
        if isinstance(n_symbols, bool) or not isinstance(n_symbols, int) or n_symbols < 2:
            raise ValueError(f"n_symbols must be an integer >= 2 (padding + one phoneme), got {n_symbols!r}")
        self.n_symbols = n_symbols
        self.embed = nn.Embedding(n_symbols, EMB, padding_idx=0)
        self.key_conv1 = nn.Conv1d(EMB, HID, 3, padding=1)
        self.key_conv2 = nn.Conv1d(HID, ATT, 1)
        self.query_conv1 = nn.Conv1d(N_MELS, 2 * N_MELS, 3, padding=1)
        self.query_conv2 = nn.Conv1d(2 * N_MELS, N_MELS, 1)
        self.query_conv3 = nn.Conv1d(N_MELS, ATT, 1)
        relu = nn.init.calculate_gain("relu")
        for conv, gain in ((self.key_conv1, relu), (self.key_conv2, 1.0), (self.query_conv1, relu), (self.query_conv2, relu),
                           (self.query_conv3, 1.0)):
            nn.init.xavier_uniform_(conv.weight, gain=gain)          # FastPitch's ConvNorm initialisation

    @staticmethod
    def _inputs(xs, ilens, mels, olens):
        if not (torch.is_tensor(xs) and xs.dim() == 2 and not xs.dtype.is_floating_point and xs.shape[1] >= 1):
            raise ValueError("xs must be a [B, T] integer tensor")
        if not (torch.is_tensor(mels) and mels.dim() == 3 and mels.shape[2] == N_MELS and mels.dtype == torch.float32):
            raise ValueError(f"mels must be a [B, L, {N_MELS}] float32 tensor")
        B, T = xs.shape
        if mels.shape[0] != B:
            raise ValueError(f"mels has {mels.shape[0]} utterances, xs {B}")
        if T > _lib.FS2_ALIGN_MAX_T:
            raise ValueError(f"T = {T} phonemes exceeds the aligner's {_lib.FS2_ALIGN_MAX_T}")
        for name, t in (("ilens", ilens), ("olens", olens)):
            if not (torch.is_tensor(t) and t.shape == (B,) and not t.dtype.is_floating_point):
                raise ValueError(f"{name} must be a [B={B}] integer tensor")
        dev = xs.device
        if dev.type != "cuda" or any(t.device != dev for t in (ilens, mels, olens)):
            raise ValueError("inputs must be CUDA tensors on one device (the aligner has no CPU path)")
        return xs.to(torch.int64).contiguous(), ilens.to(torch.int64).contiguous(), mels.contiguous(), olens.to(torch.int64).contiguous()

    def keys_queries(self, xs, ilens, mels, olens, deterministic: bool = False):
        """(k [B, T, 80], q [B, L, 80]) on the library's kernels, differentiable in the parameters.  `deterministic`: the
        embedding and bias gradients are summed in a fixed order (the deterministic train mode, DESIGN.md §26)."""
        tf32, relu, none = _lib.MATH_TF32, _train.ACT_RELU, _train.ACT_NONE
        B, T = xs.shape
        zero = torch.zeros((1,), dtype=torch.float32, device=xs.device)
        det = bool(deterministic)
        tf32 = _train.conv_math(tf32, det)
        h = _train.EmbedFn.apply(xs, self.embed.weight, zero, torch.zeros((T, EMB), dtype=torch.float32, device=xs.device), det)
        h = _train.ConvFn.apply(MaskRowsFn.apply(h, ilens), self.key_conv1.weight, self.key_conv1.bias, relu, None, tf32)
        k = _train.ConvFn.apply(MaskRowsFn.apply(h, ilens), self.key_conv2.weight, self.key_conv2.bias, none, None, tf32)
        m = _train.ConvFn.apply(MaskRowsFn.apply(mels, olens), self.query_conv1.weight, self.query_conv1.bias, relu, None, tf32)
        m = _train.ConvFn.apply(MaskRowsFn.apply(m, olens), self.query_conv2.weight, self.query_conv2.bias, relu, None, tf32)
        q = _train.ConvFn.apply(MaskRowsFn.apply(m, olens), self.query_conv3.weight, self.query_conv3.bias, none, None, tf32)
        return k, q

    def loss(self, xs, ilens, mels, olens, bin_weight: float = 0.0, deterministic: bool = False):
        """(loss, forward-sum mean, bin mean or None, status): the batch means of the per-utterance losses, loss =
        forward-sum + bin_weight * bin (the binarization loss and its MAS are skipped when bin_weight is 0).  status is
        an int32 device tensor of the entries' status words; nothing is read back to the host.  `deterministic`: see
        keys_queries (also on whenever torch.are_deterministic_algorithms_enabled())."""
        xs, ilens, mels, olens = self._inputs(xs, ilens, mels, olens)
        status = torch.zeros((7,), dtype=torch.int32, device=xs.device)
        det = bool(deterministic) or torch.are_deterministic_algorithms_enabled()
        k, q = self.keys_queries(xs, ilens, mels, olens, det)
        logp = AlignLogProbFn.apply(q, k, ilens, olens, status)
        fs = ForwardSumFn.apply(logp, ilens, olens, status).mean()
        if not bin_weight:
            return fs, fs, None, status
        with torch.no_grad():
            _, path = mas(logp.detach(), ilens, olens, status)
        bl = BinLossFn.apply(logp, path, ilens, olens, status).mean()
        return fs + float(bin_weight) * bl, fs, bl, status

    @torch.no_grad()
    def durations(self, xs, ilens, mels, olens):
        """(durations [B, T] int64, status bits): MAS durations of every utterance, each >= 1 for its phonemes and summing
        to olens[b]; an utterance flagged in status (describe_status) comes out as zeros.  Utterance b is bit-identical
        to its B = 1 call.  One host read (the status)."""
        xs, ilens, mels, olens = self._inputs(xs, ilens, mels, olens)
        status = torch.zeros((7,), dtype=torch.int32, device=xs.device)
        k, q = self.keys_queries(xs, ilens, mels, olens)
        logp = AlignLogProbFn.apply(q, k, ilens, olens, status)
        dur, _ = mas(logp, ilens, olens, status)
        return dur, status_bits(status)


# ---- training and extraction -----------------------------------------------------------------------------------------
class Corpus:
    """Filelist lines with their phoneme ids and mel frame counts; mels are read from disk per batch, or taken from
    `mels` (id -> [L, 80] array) when given."""

    def __init__(self, lines: Sequence[Line], symbols: Sequence[str], data_dir: Optional[str] = None, mels: Optional[dict] = None,
                 log=print):
        self.data_dir, self.mels = data_dir, mels
        self.lines, self.ids, self.frames, self.skipped = [], [], [], []
        for ln in lines:
            n = self._mel(ln).shape[0] if mels is not None else np.load(os.path.join(data_dir, "mels", ln.id + ".npy"), mmap_mode="r").shape[1]
            if n < len(ln.phonemes):
                log(f"skipping {ln.wav}: {len(ln.phonemes)} phonemes but {n} frames")
                self.skipped.append(ln)
                continue
            if len(ln.phonemes) > _lib.FS2_ALIGN_MAX_T:
                log(f"skipping {ln.wav}: {len(ln.phonemes)} phonemes, more than the aligner's {_lib.FS2_ALIGN_MAX_T}")
                self.skipped.append(ln)
                continue
            self.lines.append(ln)
            self.ids.append(encode(ln, symbols))
            self.frames.append(n)

    def _mel(self, ln: Line) -> np.ndarray:
        return self.mels[ln.id] if self.mels is not None else load_mel(self.data_dir, ln)

    def batch(self, idx: Sequence[int], device):
        """(xs [B, T], ilens, mels [B, L, 80], olens) on `device`, zero padded."""
        il = [len(self.ids[i]) for i in idx]
        ol = [self.frames[i] for i in idx]
        xs = np.zeros((len(idx), max(il)), np.int64)
        mels = np.zeros((len(idx), max(ol), N_MELS), np.float32)
        for j, i in enumerate(idx):
            xs[j, : il[j]] = self.ids[i]
            mels[j, : ol[j]] = self._mel(self.lines[i])
        t = lambda a: torch.from_numpy(a).to(device)
        return t(xs), t(np.array(il, np.int64)), t(mels), t(np.array(ol, np.int64))


def train(corpus: Corpus, n_symbols: int, steps: int, batch: int = 32, bin_start: Optional[int] = None, seed: int = 0,
          warmup: int = 4000, factor: float = 1.0, grad_clip: float = 1.0, device="cuda", log=print, log_every: int = 100,
          deterministic: bool = False):
    """Trains an Aligner for `steps` steps of `batch` utterances (length-bucketed) with NoamAdam(model size 256, factor,
    warmup), clipping at grad_clip; the binarization loss is weighted 1 from step bin_start on (default steps // 2).
    `deterministic` (or torch.use_deterministic_algorithms(True)): every gradient is summed in a fixed order, so the same
    corpus and seed give the same weights bit for bit (DESIGN.md §26).
    Returns (model, [(step, loss, forward-sum, bin or None)] at every log_every-th step)."""
    if not corpus.lines:
        raise ValueError("no trainable lines in the corpus")
    torch.manual_seed(seed)
    model = Aligner(n_symbols).to(device)
    opt = NoamAdam(model.parameters(), EMB, factor, warmup)
    bin_start = steps // 2 if bin_start is None else bin_start
    sampler = BucketBatchSampler(corpus.frames, min(batch, len(corpus.lines)), seed=seed)
    history, step, epoch = [], 0, 0
    while step < steps:
        sampler.set_epoch(epoch)
        for idx in sampler:
            if step >= steps:
                break
            loss, fs, bl, status = model.loss(*corpus.batch(idx, device), bin_weight=1.0 if step >= bin_start else 0.0,
                                              deterministic=deterministic)
            opt.zero_grad()
            loss.backward()
            opt.clip_and_step(grad_clip)
            step += 1
            if step % log_every == 0 or step == steps:
                bits = status_bits(status)
                if bits:
                    raise RuntimeError(f"aligner step {step}: {describe_status(bits)}")
                rec = (step, float(loss), float(fs), None if bl is None else float(bl))
                history.append(rec)
                log(json.dumps({"step": step, "loss": rec[1], "forward_sum": rec[2], "bin": rec[3]}))
        epoch += 1
    return model, history


def extract(model: Aligner, corpus: Corpus, batch: int = 32, device="cuda") -> List[np.ndarray]:
    """MAS durations of every line of the corpus, in corpus order."""
    out: List[Optional[np.ndarray]] = [None] * len(corpus.lines)
    order = np.argsort(corpus.frames, kind="stable")
    for s in range(0, len(order), batch):
        idx = order[s: s + batch].tolist()
        xs, ilens, mels, olens = corpus.batch(idx, device)
        dur, bits = model.durations(xs, ilens, mels, olens)
        if bits:
            raise RuntimeError(f"aligner extraction: {describe_status(bits)}")
        dur = dur.cpu().numpy()
        for j, i in enumerate(idx):
            out[i] = dur[j, : len(corpus.ids[i])]
    return out


def agreement(lines: Sequence[Line], durations: Sequence[np.ndarray]) -> Optional[dict]:
    """Agreement of `durations` with the durations the lines carry: fraction of phonemes within 1 and 2 frames, mean
    absolute difference of the phoneme end frames, and the file where that mean is worst.  None when no line has any."""
    diffs, bounds, worst = [], [], (-1.0, None)
    for ln, d in zip(lines, durations):
        if ln.durations is None:
            continue
        ref = np.asarray(ln.durations, np.int64)
        diffs.append(np.abs(np.asarray(d) - ref))
        b = np.abs(np.cumsum(d) - np.cumsum(ref))
        bounds.append(b)
        if b.mean() > worst[0]:
            worst = (float(b.mean()), ln.wav)
    if not diffs:
        return None
    dd, bb = np.concatenate(diffs), np.concatenate(bounds)
    return {"lines": len(diffs), "phonemes": int(dd.size), "within_1": float((dd <= 1).mean()), "within_2": float((dd <= 2).mean()),
            "mean_abs_boundary_frames": float(bb.mean()), "worst_file": worst[1], "worst_mean_abs_boundary_frames": worst[0]}


def save(path: str, model: Aligner, symbols: Sequence[str], step: int) -> None:
    torch.save({"model": {k: v.detach().cpu() for k, v in model.state_dict().items()}, "symbols": list(symbols), "step": int(step)}, path)


def load(path: str, device="cuda"):
    """(model, symbols, step) from a checkpoint written by `save`."""
    ck = torch.load(path, map_location="cpu", weights_only=True)
    if not isinstance(ck, dict) or not {"model", "symbols", "step"} <= set(ck):
        raise ValueError(f"{path}: not an aligner checkpoint (needs model, symbols and step)")
    symbols = list(ck["symbols"])
    model = Aligner(len(symbols))
    model.load_state_dict(ck["model"], strict=True)
    return model.to(device), symbols, int(ck["step"])


def _data_dir(args, hp) -> str:
    if args.data_dir:
        return args.data_dir
    data = hp.get("data", {}) if isinstance(hp, dict) else {}
    if not data.get("data_dir"):
        raise SystemExit("no data directory: pass -d or set data.data_dir in the config")
    return data["data_dir"]


def main(argv=None) -> None:
    from .hparams import load_hp
    ap = argparse.ArgumentParser(prog="python -m fastspeech2_b200.aligner", description=__doc__.split("\n\n")[0])
    sub = ap.add_subparsers(dest="cmd", required=True)
    for name in ("train", "extract"):
        p = sub.add_parser(name)
        p.add_argument("-c", "--config", required=True, help="yaml file for configuration")
        p.add_argument("--filelist", required=True, help="filelist in the reference's five-field format")
        p.add_argument("-d", "--data_dir", default=None, help="preprocess output directory (default: data.data_dir of the config)")
        p.add_argument("--batch", type=int, default=32, help="utterances per batch")
    t = sub.choices["train"]
    t.add_argument("--steps", type=int, default=20000)
    t.add_argument("--bin-start", type=int, default=None, help="step from which the binarization loss is on (default: steps / 2)")
    t.add_argument("-o", "--out", required=True, help="checkpoint to write")
    t.add_argument("--deterministic", action="store_true",
                   help="sum every gradient in a fixed order, so a rerun gives the same checkpoint bit for bit")
    e = sub.choices["extract"]
    e.add_argument("-p", "--checkpoint", required=True, help="aligner checkpoint written by train")
    e.add_argument("--out", required=True, help="filelist to write")
    args = ap.parse_args(argv)
    if args.batch < 1 or (args.cmd == "train" and args.steps < 1):
        ap.error("--batch and --steps must be positive")
    hp = load_hp(args.config)
    data_dir = _data_dir(args, hp)
    lines = read_filelist(args.filelist)
    if args.cmd == "train":
        symbols = build_symbols(lines)
        corpus = Corpus(lines, symbols, data_dir, log=lambda m: print(m, file=sys.stderr))
        model, _ = train(corpus, len(symbols), args.steps, args.batch, args.bin_start, deterministic=args.deterministic)
        save(args.out, model, symbols, args.steps)
        return
    model, symbols, _ = load(args.checkpoint)
    corpus = Corpus(lines, symbols, data_dir, log=lambda m: print(m, file=sys.stderr))
    durs = extract(model, corpus, args.batch)
    with open(args.out, "w", encoding="utf-8") as fh:
        for ln, d in zip(corpus.lines, durs):
            fh.write(format_line(ln, d) + "\n")
    agr = agreement(corpus.lines, durs)
    if agr is not None:
        print(json.dumps(agr))


if __name__ == "__main__":
    main()
