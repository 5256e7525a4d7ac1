"""Input side of the path (SURVEY.md section 8f-3): batch assembly with the reference's tensor contract.

* `collate_tts(batch)` -- same 9-tuple as the reference's dataset/dataloader.py:96-118
  (inputs, ilens, mels, labels, olens, ids, durations, energys, pitches), zero padded to the batch maxima.
* `PinnedCollator` -- the same tensors assembled straight into reusable page-locked buffers, so the seven H2D
  copies the reference issues per step (train_fastspeech.py:101-107) become asynchronous `non_blocking` copies.
* `BucketBatchSampler` -- length-bucketed batches.  The forward path computes the whole padded [B, Lmax] rectangle
  (the reference's convolutions read padded frames, SURVEY.md section 0), so padding is real work: bucketing by
  mel length cuts it.  (The reference ships a BinnedLengthSampler, dataloader.py:121-150, but never instantiates it.)

Items are the reference's `TTSDataset.__getitem__` tuples (dataloader.py:47-74):
  (phoneme ids [T] int, mel [L, n_mels] float, id str, mel_len int, durations [T] int, energy [L] float, pitch [L] float),
optionally followed by an 8th element, the speaker id (multi-speaker models, DESIGN.md section 25).  When every item of a
batch has it, `collate_tts` and `PinnedCollator` return a 10th element, speakers [B] int64; with 7-element items the
9-tuple is unchanged.  A 9th element is the utterance's speaker embedding, float32 [D] (models with spk_embed_dim,
DESIGN.md section 27), after the speaker id or None when there is no speaker table; when every item has it, the 10th
element is speakers [B] int64 or None, and an 11th follows, spembs [B, D] float32.  `FilelistDataset` reads such items
from a `preprocess` tree.
"""
from __future__ import annotations

import os
from typing import Dict, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch


def _lens(batch) -> Tuple[List[int], List[int]]:
    return [int(np.shape(it[0])[0]) for it in batch], [int(np.shape(it[1])[0]) for it in batch]


def _speakers(batch) -> Optional[List[int]]:
    """The batch's speaker ids (8th item element), or None when the items have 7 elements (or 9 with None there)."""
    n = {len(it) for it in batch}
    if n == {7}:
        return None
    if n not in ({8}, {9}):
        raise ValueError(f"items must all have 7 elements, all 8 (with the speaker id) or all 9 (speaker id or None, then the "
                         f"speaker embedding); got lengths {sorted(n)}")
    if n == {9} and all(it[7] is None for it in batch):
        return None
    if any(it[7] is None for it in batch):
        raise ValueError("items must all carry a speaker id or all carry None")
    return [int(it[7]) for it in batch]


def _spembs(batch) -> Optional[np.ndarray]:
    """The batch's speaker embeddings (9th item element) as float32 [B, D], or None when the items have fewer elements."""
    if len(batch[0]) != 9:
        return None
    out = [np.asarray(it[8], dtype=np.float32) for it in batch]
    shapes = {e.shape for e in out}
    if len(shapes) != 1 or len(next(iter(shapes))) != 1:
        raise ValueError(f"speaker embeddings must all be [D] with one D, got shapes {sorted(shapes)}")
    return np.stack(out)


def _fill(batch, inputs, mels, durations, energys, pitches, labels):
    for i, it in enumerate(batch):
        x, mel, dur, e, p = (torch.as_tensor(np.asarray(it[k])) for k in (0, 1, 4, 5, 6))
        T, L = x.shape[0], mel.shape[0]
        inputs[i, :T] = x
        mels[i, :L] = mel
        durations[i, : dur.shape[0]] = dur
        energys[i, : e.shape[0]] = e
        pitches[i, : p.shape[0]] = p
        labels[i, L - 1:] = 1.0          # stop-token labels, dataloader.py:110-112


def collate_tts(batch: Sequence[tuple]):
    """Drop-in for the reference's `collate_tts`."""
    il, ol = _lens(batch)
    B, T, L = len(batch), max(il), max(ol)
    n_mels = int(np.shape(batch[0][1])[1])
    Td = max(int(np.shape(it[4])[0]) for it in batch)
    Le, Lp = max(int(np.shape(it[5])[0]) for it in batch), max(int(np.shape(it[6])[0]) for it in batch)
    inputs = torch.zeros(B, T, dtype=torch.int64)
    mels = torch.zeros(B, L, n_mels, dtype=torch.float32)
    durations = torch.zeros(B, Td, dtype=torch.int64)
    energys = torch.zeros(B, Le, dtype=torch.float32)
    pitches = torch.zeros(B, Lp, dtype=torch.float32)
    labels = torch.zeros(B, L, dtype=torch.float32)
    _fill(batch, inputs, mels, durations, energys, pitches, labels)
    ids = [it[2] for it in batch]
    out = (inputs, torch.tensor(il, dtype=torch.int64), mels, labels, torch.tensor(ol, dtype=torch.int64), ids, durations, energys, pitches)
    spk = _speakers(batch)
    spe = _spembs(batch)
    spk_t = None if spk is None else torch.tensor(spk, dtype=torch.int64)
    if spe is not None:
        return out + (spk_t, torch.from_numpy(spe))
    return out if spk is None else out + (spk_t,)


class _Collated(tuple):
    """The 9-tuple of `collate_tts` plus the pinned slot it lives in."""
    slot = -1


class PinnedCollator:
    """`collate_tts` into reusable pinned host buffers + asynchronous upload.

    `collator(batch)` returns the 9-tuple with pinned CPU tensors (views of one of `slots` buffer sets);
    `collator.to_device(tuple, device)` issues the H2D copies with `non_blocking=True` on the current stream and records a
    CUDA event for that slot.  Before a slot is refilled its event is waited for, so a loader that runs ahead of the GPU
    can never overwrite host memory an earlier asynchronous copy is still reading (with `slots` batches in flight).
    """

    def __init__(self, max_batch: int, max_T: int, max_L: int, n_mels: int = 80, pin: Optional[bool] = None, slots: int = 2,
                 spk_embed_dim: int = 0):
        pin = torch.cuda.is_available() if pin is None else pin
        mk = lambda shape, dt: torch.zeros(shape, dtype=dt).pin_memory() if pin else torch.zeros(shape, dtype=dt)
        self.cap = (max_batch, max_T, max_L)
        self.n_mels = n_mels
        self.slots = [dict(inputs=mk((max_batch, max_T), torch.int64), durations=mk((max_batch, max_T), torch.int64),
                           mels=mk((max_batch, max_L, n_mels), torch.float32), labels=mk((max_batch, max_L), torch.float32),
                           energys=mk((max_batch, max_L), torch.float32), pitches=mk((max_batch, max_L), torch.float32),
                           ilens=mk((max_batch,), torch.int64), olens=mk((max_batch,), torch.int64),
                           speakers=mk((max_batch,), torch.int64), event=None,
                           spembs=mk((max_batch, spk_embed_dim), torch.float32) if spk_embed_dim else None)
                      for _ in range(max(1, int(slots)))]
        self.spk_embed_dim = int(spk_embed_dim)
        self._next = 0

    def __call__(self, batch: Sequence[tuple]):
        il, ol = _lens(batch)
        B, T, L = len(batch), max(il), max(ol)
        if B > self.cap[0] or T > self.cap[1] or L > self.cap[2]:
            raise ValueError(f"batch {B}x{T}x{L} exceeds the pinned capacity {self.cap}")
        idx = self._next
        self._next = (idx + 1) % len(self.slots)
        s = self.slots[idx]
        if s["event"] is not None:          # the upload that last read this slot must have finished
            s["event"].synchronize()
            s["event"] = None
        # dense [B, T] / [B, L] windows of the big buffers are not contiguous; stage into contiguous prefixes instead
        n_mels = self.n_mels
        inputs = s["inputs"].view(-1)[: B * T].view(B, T).zero_()
        durations = s["durations"].view(-1)[: B * T].view(B, T).zero_()
        mels = s["mels"].view(-1)[: B * L * n_mels].view(B, L, n_mels).zero_()
        labels = s["labels"].view(-1)[: B * L].view(B, L).zero_()
        energys = s["energys"].view(-1)[: B * L].view(B, L).zero_()
        pitches = s["pitches"].view(-1)[: B * L].view(B, L).zero_()
        _fill(batch, inputs, mels, durations, energys, pitches, labels)
        ilens, olens = s["ilens"][:B], s["olens"][:B]
        ilens.copy_(torch.tensor(il)); olens.copy_(torch.tensor(ol))
        items = (inputs, ilens, mels, labels, olens, [it[2] for it in batch], durations, energys, pitches)
        spk = _speakers(batch)
        spe = _spembs(batch)
        speakers = None
        if spk is not None:
            speakers = s["speakers"][:B]
            speakers.copy_(torch.tensor(spk, dtype=torch.int64))
        if spe is not None:
            if spe.shape[1] != self.spk_embed_dim:
                raise ValueError(f"speaker embeddings of D={spe.shape[1]}, but the collator holds spk_embed_dim={self.spk_embed_dim}")
            spembs = s["spembs"][:B]
            spembs.copy_(torch.from_numpy(spe))
            items = items + (speakers, spembs)
        elif speakers is not None:
            items = items + (speakers,)
        out = _Collated(items)
        out.slot = idx
        return out

    def to_device(self, collated, device):
        """Asynchronous H2D of every tensor of `collated` on the current stream of `device`; remembers an event so the
        slot is not refilled before the copies have run."""
        out = tuple(t.to(device, non_blocking=True) if torch.is_tensor(t) else t for t in collated)
        slot = getattr(collated, "slot", -1)
        if slot >= 0 and torch.device(device).type == "cuda":
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(device))
            self.slots[slot]["event"] = ev
        return out

    def upload_into(self, collated, dst: Sequence[Optional[torch.Tensor]]):
        """Like `to_device`, but copies into existing device tensors (e.g. the static inputs of a captured CUDA graph):
        `dst[i]` receives `collated[i]` (None / non-tensor entries are skipped).  Asynchronous, same slot bookkeeping."""
        dev = None
        for src, d in zip(collated, dst):
            if d is not None and torch.is_tensor(src):
                d.copy_(src, non_blocking=True)
                dev = d.device
        slot = getattr(collated, "slot", -1)
        if slot >= 0 and dev is not None and dev.type == "cuda":
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(dev))
            self.slots[slot]["event"] = ev


class BucketBatchSampler:
    """Batches of indices with similar length: sort by length, cut into bins of `bin_size`, shuffle inside and
    across bins with a seeded generator, then chunk into batches.  `padding_waste(lengths)` reports the fraction
    of padded positions the resulting batches contain (what the rectangle computation pays for)."""

    def __init__(self, lengths: Sequence[int], batch_size: int, bin_size: Optional[int] = None, seed: int = 0, drop_last: bool = False):
        self.lengths = torch.as_tensor(list(lengths), dtype=torch.int64)
        self.batch_size = int(batch_size)
        self.bin_size = int(bin_size or 8 * batch_size)
        if self.bin_size % self.batch_size:
            raise ValueError("bin_size must be a multiple of batch_size")
        self.seed, self.epoch, self.drop_last = seed, 0, drop_last

    def set_epoch(self, epoch: int) -> None:
        self.epoch = epoch

    def __iter__(self) -> Iterator[List[int]]:
        g = torch.Generator().manual_seed(self.seed + self.epoch)
        order = torch.argsort(self.lengths, stable=True)
        bins = [order[i: i + self.bin_size] for i in range(0, len(order), self.bin_size)]
        bins = [b[torch.randperm(len(b), generator=g)] for b in bins]
        batches: List[List[int]] = []
        for b in bins:
            for i in range(0, len(b), self.batch_size):
                chunk = b[i: i + self.batch_size].tolist()
                if len(chunk) == self.batch_size or not self.drop_last:
                    batches.append(chunk)
        for i in torch.randperm(len(batches), generator=g).tolist():
            yield batches[i]

    def __len__(self) -> int:
        n = len(self.lengths)
        return n // self.batch_size if self.drop_last else (n + self.batch_size - 1) // self.batch_size

    def padding_waste(self) -> float:
        pad = tot = 0
        for batch in self:
            ls = self.lengths[batch]
            tot += int(ls.max()) * len(batch)
            pad += int(ls.max()) * len(batch) - int(ls.sum())
        return pad / max(tot, 1)


class FilelistDataset:
    """The reference's `TTSDataset` (dataloader.py:34-74) on a `preprocess` tree, plus the speaker id and embedding.

    `filelist`: 5- or 6-field lines (aligner.parse_line); `data_dir`: holds mels/, energy/ and pitch/{id}.npy;
    `symbols`: the phoneme table (aligner.build_symbols -- the reference's 68-symbol table belongs to its text front-end);
    `speaker_map` ({name: id}, speakers.build_map / load_map) or None for a single-speaker corpus.  Item i is
    (phoneme ids, mel [L, n_mels], id, L, durations, energy, pitch[, speaker id]) with the reference loader's corrections:
    durations cut to the phonemes and the last one stretched so that they sum to L, remove_outlier on energy and pitch.
    `spemb_dir` (DESIGN.md section 27): a directory of `{id}.npy` speaker embeddings, one float32 [D] per utterance (id =
    the wav name up to its first dot), from any extractor; items then carry it as a 9th element, after the speaker id or
    None."""

    def __init__(self, filelist: str, data_dir: str, symbols: Sequence[str], speaker_map: Optional[Dict[str, int]] = None,
                 spemb_dir: Optional[str] = None):
        from .aligner import read_filelist
        self.lines = read_filelist(filelist)
        self.data_dir = data_dir
        self.table = {s: i for i, s in enumerate(symbols)}
        self.speaker_map = speaker_map
        self.spemb_dir = spemb_dir
        for ln in self.lines:
            if ln.durations is None:
                raise ValueError(f"{ln.wav}: no durations (run `python -m fastspeech2_b200.aligner extract` first)")
        if speaker_map is not None:
            from .speakers import speaker_of
            missing = sorted({speaker_of(ln) for ln in self.lines} - set(speaker_map))
            if missing:
                raise ValueError(f"speakers {missing[:5]} are not in the speaker map")

    def __len__(self) -> int:
        return len(self.lines)

    def __getitem__(self, index: int) -> tuple:
        from .aligner import encode
        from .preprocess import remove_outlier
        ln = self.lines[index]
        x = encode(ln, list(self.table))
        path = lambda kind: os.path.join(self.data_dir, kind, ln.id + ".npy")
        mel = np.load(path("mels"))
        L = int(mel.shape[1])
        d = list(ln.durations)[: len(x)]
        d[-1] = d[-1] + (L - sum(d))                       # dataloader.py:64-65
        if d[-1] < 0:
            raise ValueError(f"{ln.wav}: durations sum past the mel's {L} frames")
        e = remove_outlier(np.load(path("energy")))
        p = remove_outlier(np.load(path("pitch")))
        item = (x, mel.T, ln.id, L, np.array(d, dtype=np.int64), e, p)
        spk = None
        if self.speaker_map is not None:
            from .speakers import speaker_of
            spk = self.speaker_map[speaker_of(ln)]
        if self.spemb_dir is None:
            return item if spk is None else item + (spk,)
        return item + (spk, load_spemb(os.path.join(self.spemb_dir, ln.id + ".npy")))

    def spemb_dim(self) -> int:
        """D of the first utterance's embedding (spemb_dir given), else 0."""
        if self.spemb_dir is None or not self.lines:
            return 0
        return int(load_spemb(os.path.join(self.spemb_dir, self.lines[0].id + ".npy")).shape[0])

    def mel_lengths(self) -> List[int]:
        """Frames per item (BucketBatchSampler's lengths), read from the mel files' headers."""
        return [int(np.load(os.path.join(self.data_dir, "mels", ln.id + ".npy"), mmap_mode="r").shape[1]) for ln in self.lines]


def load_spemb(path: str) -> np.ndarray:
    """One speaker embedding file: a [D] (or [1, D]) array of any float dtype -> float32 [D]."""
    e = np.load(path)
    if e.ndim == 2 and e.shape[0] == 1:
        e = e[0]
    if e.ndim != 1 or e.shape[0] < 1 or not np.issubdtype(e.dtype, np.floating):
        raise ValueError(f"{path}: a speaker embedding must be a float [D] array, got {e.dtype} {e.shape}")
    return e.astype(np.float32)
