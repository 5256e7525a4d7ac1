"""Data-parallel synthesis over the GPUs of one box (SURVEY.md section 8e).

Utterances are independent, so the batch is cut into contiguous shards, one process per GPU, weights
replicated.  The path has exactly one exchange step: the all-gather of the final mel shards (plus
their lengths).  When shards have different padded lengths a tiny all-reduce(max) of Lmax comes
first so every rank contributes a `[B_r, Lmax, odim]` block.

Works with any torch.distributed backend: NCCL over NVLink on the GPU box, gloo on CPU for the
host-logic tests (tests/test_sharded_gloo.py).
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.distributed as dist


def shard_bounds(n_items: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous block of `n_items` owned by `rank`: sizes differ by at most one, earlier ranks larger."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def gather_mels(mel: torch.Tensor, olens: torch.Tensor, group: Optional[dist.ProcessGroup] = None,
                equal_shapes: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """All-gather `[B_r, L_r, odim]` mel shards (zero-extended to the global Lmax) and `[B_r]` lengths.

    Returns (`[sum B_r, Lmax, odim]`, `[sum B_r]`) on every rank, in rank order.  `equal_shapes=True`
    skips the shape exchange (the benchmark's equal shards): a single collective on the mels.
    """
    world = dist.get_world_size(group)
    if world == 1:
        return mel, olens
    B, L, D = mel.shape
    if equal_shapes:
        out = torch.empty((world * B, L, D), dtype=mel.dtype, device=mel.device)
        dist.all_gather_into_tensor(out, mel.contiguous(), group=group)
        lens = torch.empty((world * B,), dtype=olens.dtype, device=olens.device)
        dist.all_gather_into_tensor(lens, olens.contiguous(), group=group)
        return out, lens
    shape = torch.tensor([B, L], dtype=torch.int64, device=mel.device)
    shapes = [torch.empty_like(shape) for _ in range(world)]
    dist.all_gather(shapes, shape, group=group)
    shapes = [tuple(int(v) for v in s.tolist()) for s in shapes]
    Lmax = max(s[1] for s in shapes)
    Bmax = max(s[0] for s in shapes)
    block = torch.zeros((Bmax, Lmax, D), dtype=mel.dtype, device=mel.device)
    block[:B, :L] = mel
    lens_block = torch.zeros((Bmax,), dtype=olens.dtype, device=olens.device)
    lens_block[:B] = olens
    blocks = torch.empty((world, Bmax, Lmax, D), dtype=mel.dtype, device=mel.device)
    dist.all_gather_into_tensor(blocks.view(world * Bmax, Lmax, D), block, group=group)
    lens_all = torch.empty((world * Bmax,), dtype=olens.dtype, device=olens.device)
    dist.all_gather_into_tensor(lens_all, lens_block, group=group)
    mels = torch.cat([blocks[r, : shapes[r][0]] for r in range(world)], dim=0)
    lens = torch.cat([lens_all[r * Bmax: r * Bmax + shapes[r][0]] for r in range(world)], dim=0)
    return mels, lens


def gather_mels_to_root(mel: torch.Tensor, dst: int = 0, group: Optional[dist.ProcessGroup] = None,
                        out: Optional[torch.Tensor] = None) -> Optional[torch.Tensor]:
    """Gather equal-shape `[B, L, odim]` mel shards on rank `dst` only (the other ranks just send their 1/N share):
    the "gather of the final mel batch" of SURVEY section 8e without the N-fold fan-out of an all-gather.  Returns the
    `[world*B, L, odim]` batch on `dst` (written into `out` when given) and None elsewhere."""
    world = dist.get_world_size(group)
    if world == 1:
        return mel
    B, L, D = mel.shape
    rank = dist.get_rank(group)
    if rank == dst:
        if out is None:
            out = torch.empty((world * B, L, D), dtype=mel.dtype, device=mel.device)
        dist.gather(mel.contiguous(), list(out.view(world, B, L, D).unbind(0)), dst=dst, group=group)
        return out
    dist.gather(mel.contiguous(), None, dst=dst, group=group)
    return None


class _RawCudaBuffer:
    """Zero-copy tensor view of a raw device pointer (local cudaMalloc or a peer's IPC mapping)."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (int(ptr), False), "version": 2}


class PeerGather:
    """Gather-to-root of equal-shape `[B, L, odim]` mel shards over NVLink peer memory (csrc/peer.cu): one copy-engine
    transfer per rank and step on a side stream, flag words for completion, no NCCL kernel on the SMs.

        pg = PeerGather((B, L, odim), device)            # collective: every rank of the group calls it once
        pg.push(mel, step)                               # every rank, after its step's mel is complete on the current stream
        pg.wait(step)                                    # root: later work on the current stream sees all shards of `step`
        pg.gathered                                      # root: [world*B, L, odim] view of the receive buffer

    `push` returns immediately (the transfer runs on `pg.stream`); the source tensor must stay untouched until
    `pg.pushed` (an event recorded after the transfer) has completed.  With a non-CUDA tensor (gloo host-logic tests) the
    class degrades to `gather_mels_to_root`.

    Fused form (no transfer at all): `pg.slot(i)` is this rank's shard of receive buffer `i` as a tensor -- on non-root
    ranks a view of the ROOT's memory mapped over NVLink.  Passed as the output of the last Postnet kernel
    (`model.graphed_forward(..., after_out=pg.slot(i))`), that kernel's epilogue stores the mels straight into the root's
    buffer tile by tile while it computes; `pg.signal(step)` then publishes the step with one flag store.  `buffers` > 1
    gives that many receive buffers (alternating CUDA graphs write alternating buffers)."""

    HEADER = 256          # bytes reserved for the flag words in front of the shards

    def __init__(self, shard_shape, device, dtype=torch.float32, root: int = 0, group: Optional[dist.ProcessGroup] = None, buffers: int = 1):
        self.group, self.root, self.buffers, self.dtype = group, root, max(1, int(buffers)), dtype
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.shape = tuple(int(v) for v in shard_shape)
        self.device = torch.device(device)
        self.gathered = None
        self.pushed = None
        self._cuda = self.device.type == "cuda"
        if not self._cuda or self.world == 1:
            return
        import ctypes as C
        from . import _lib
        self._lib = _lib.load()
        n = 1
        for v in self.shape:
            n *= v
        self.shard_bytes = n * torch.empty((), dtype=dtype).element_size()
        total = self.HEADER + self.buffers * self.world * self.shard_bytes
        assert self.world * 8 <= self.HEADER
        handle = (C.c_char * 64)()
        ptr = C.c_void_p()
        err = None
        with torch.cuda.device(self.device):
            # every rank takes part in every collective below whatever fails locally, then all agree on success
            if self.rank == root:
                try:
                    _lib.check(self._lib.fs2_peer_alloc(total, C.byref(ptr), handle), "fs2_peer_alloc")
                except Exception as e:          # noqa: BLE001
                    err = e
            obj = [bytes(handle) if (self.rank == root and err is None) else None]
            dist.broadcast_object_list(obj, src=root, group=group, device=self.device)
            if self.rank != root:
                try:
                    if obj[0] is None:
                        raise _lib.Fs2Error("the root rank could not export its receive buffer")
                    _lib.check(self._lib.fs2_peer_open(C.create_string_buffer(obj[0], 64), C.byref(ptr)), "fs2_peer_open")
                except Exception as e:          # noqa: BLE001
                    err = e
            ok = torch.tensor([0.0 if err is not None else 1.0], device=self.device)
            dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
        self._base = int(ptr.value or 0)
        if float(ok) < 1:
            if self._base:
                (self._lib.fs2_peer_free if self.rank == root else self._lib.fs2_peer_close)(self._base)
                self._base = 0
            raise _lib.Fs2Error(f"PeerGather: peer memory unavailable on at least one rank ({err})")
        self._flags = self._base
        self._data = self._base + self.HEADER
        self.stream = torch.cuda.Stream(self.device)
        if self.rank == root:
            raw = torch.as_tensor(_RawCudaBuffer(self._data, self.buffers * self.world * self.shard_bytes), device=self.device)
            self._all = raw.view(dtype).view((self.buffers, self.world * self.shape[0]) + self.shape[1:])
            self.gathered = self._all[0]

    def slot(self, buffer: int = 0) -> torch.Tensor:
        """This rank's shard of receive buffer `buffer` as a [B, L, odim] tensor (root: local memory; other ranks: the
        root's memory mapped over NVLink -- stores to it travel as peer writes)."""
        if not self._cuda or self.world == 1:
            raise RuntimeError("PeerGather.slot needs the CUDA / multi-rank form")
        off = self._data + (buffer * self.world + self.rank) * self.shard_bytes
        raw = torch.as_tensor(_RawCudaBuffer(off, self.shard_bytes), device=self.device)
        return raw.view(self.dtype).view(self.shape)

    def gathered_buffer(self, buffer: int = 0) -> Optional[torch.Tensor]:
        return self._all[buffer] if (self._cuda and self.world > 1 and self.rank == self.root) else self.gathered

    def signal(self, step: int) -> None:
        """Fused form: everything this rank stored into its slot on the current stream is complete -> publish `step`."""
        if not self._cuda or self.world == 1 or self.rank == self.root:
            return
        from . import _lib
        cur = torch.cuda.current_stream(self.device)
        _lib.check(self._lib.fs2_flag_signal(self._flags + 8 * self.rank, int(step), cur.cuda_stream), "fs2_flag_signal")

    def push(self, mel: torch.Tensor, step: int) -> None:
        if not self._cuda or self.world == 1:
            out = gather_mels_to_root(mel, dst=self.root, group=self.group)
            if self.rank == self.root:
                self.gathered = out
            return
        from . import _lib
        cur = torch.cuda.current_stream(self.device)
        ready = torch.cuda.Event()
        ready.record(cur)
        self.stream.wait_event(ready)
        st = self.stream.cuda_stream
        dst = self._data + self.rank * self.shard_bytes
        _lib.check(self._lib.fs2_peer_copy(dst, mel.data_ptr(), self.shard_bytes, st), "fs2_peer_copy")
        if self.rank != self.root:
            _lib.check(self._lib.fs2_flag_signal(self._flags + 8 * self.rank, int(step), st), "fs2_flag_signal")
        self.pushed = torch.cuda.Event()
        self.pushed.record(self.stream)

    def wait(self, step: int) -> None:
        """Root: order the current stream after the arrival of every rank's shard of `step` (and its own local copy)."""
        if not self._cuda or self.world == 1 or self.rank != self.root:
            return
        from . import _lib
        cur = torch.cuda.current_stream(self.device)
        if self.pushed is not None:
            cur.wait_event(self.pushed)
        _lib.check(self._lib.fs2_flag_wait(self._flags, self.world, self.root, int(step), cur.cuda_stream), "fs2_flag_wait")

    def close(self) -> None:
        if not self._cuda or self.world == 1 or self._base == 0:
            return
        torch.cuda.synchronize(self.device)
        dist.barrier(group=self.group)
        if self.rank == self.root:
            self.gathered = None
            self._lib.fs2_peer_free(self._base)
        else:
            self._lib.fs2_peer_close(self._base)
        self._base = 0


def synthesize_sharded(model, xs: torch.Tensor, ilens: torch.Tensor, group: Optional[dist.ProcessGroup] = None,
                       speakers: Optional[torch.Tensor] = None, spembs: Optional[torch.Tensor] = None):
    """Batched `is_inference=True` synthesis of a global batch: every rank passes the same global
    `xs [B,T]` / `ilens [B]` (and, for a multi-speaker model, `speakers [B]`; for a model with speaker embeddings,
    `spembs [B, D]`), runs its shard and receives all mels.
    Returns (mels, olens)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    lo, hi = shard_bounds(xs.shape[0], rank, world)
    il = ilens[lo:hi]
    t = int(il.max()) if hi > lo else 0
    with torch.no_grad():
        _, after, d_outs, _, _ = model._forward(xs[lo:hi, :t].contiguous(), il, is_inference=True, _one_hot=False,
                                                speakers=None if speakers is None else speakers[lo:hi],
                                                spembs=None if spembs is None else spembs[lo:hi])
    olens = d_outs.sum(dim=1)
    if world == 1:
        return after, olens
    return gather_mels(after, olens, group)


class GradientSync:
    """Data-parallel training step of SURVEY.md section 8f-1 (the reference itself has no data parallelism; its loop is
    `loss.backward(); clip_grad_norm_; optimizer.step()`, train_fastspeech.py:117-124): every rank runs
    `loss, report = model(...); loss.backward()` on its own utterance shard, then

        sync = GradientSync(model)          # once: flat fp32 bucket, every parameter's .grad becomes a view of it
        ...
        loss.backward()
        sync.all_reduce()                   # ONE collective over the whole bucket (NCCL ring / NVLS over NVLink), mean over ranks
        clip_grad_norm_(...); optimizer.step(); sync.zero_grad()
        # or, with fastspeech2_b200.optim.NoamAdam (the grads stay views of the bucket):
        norm = optimizer.clip_and_step(grad_clip); sync.zero_grad()

    The whole model is 35 M parameters = 141 MB of fp32 gradients: one bucket, one launch -- with NVSwitch the cost is
    launch latency plus bytes, so splitting into DDP-style 25 MB buckets buys nothing once backward has finished, and
    the backward of this model is ~100 short launches with nothing long to hide a collective behind.  Semantics are
    those of torch DDP: the mean over ranks of per-shard masked-mean losses (equal to the single-process gradient when
    shards hold the same number of valid frames / phonemes, as the bucketed sampler arranges).
    `broadcast_parameters()` makes every rank start from the root's weights (and BatchNorm running statistics).
    Backend-agnostic (gloo on CPU for the host-logic test)."""

    def __init__(self, model: torch.nn.Module, group: Optional[dist.ProcessGroup] = None):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.params = [p for p in model.parameters() if p.requires_grad]
        if not self.params:
            raise ValueError("GradientSync: the model has no trainable parameters")
        dev, dt = self.params[0].device, self.params[0].dtype
        if any(p.device != dev or p.dtype != dt for p in self.params):
            raise ValueError("GradientSync: parameters must share one device and dtype")
        self.model = model
        sizes = [p.numel() for p in self.params]
        # 128-byte aligned segments so every view is a legal vector-access target for the backward kernels
        self.offsets, off = [], 0
        for n in sizes:
            self.offsets.append(off)
            off += (n + 31) // 32 * 32
        self.flat = torch.zeros(off, dtype=dt, device=dev)
        for p, o, n in zip(self.params, self.offsets, sizes):
            view = self.flat[o:o + n].view_as(p)
            if p.grad is not None:
                view.copy_(p.grad)
            p.grad = view

    def _check_views(self) -> None:
        for p, o in zip(self.params, self.offsets):
            if p.grad is None or p.grad.data_ptr() != self.flat.data_ptr() + o * self.flat.element_size():
                raise RuntimeError("GradientSync: a parameter's .grad no longer aliases the bucket "
                                   "(use sync.zero_grad(), not optimizer.zero_grad(set_to_none=True))")

    def all_reduce(self) -> None:
        """Mean of the gradient bucket over the ranks, in place; enqueued on the current stream (NCCL) / blocking (gloo)."""
        self._check_views()
        if self.world == 1:
            return
        if self.flat.is_cuda:
            dist.all_reduce(self.flat, op=dist.ReduceOp.AVG, group=self.group)
        else:                                   # gloo has no AVG
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=self.group)
            self.flat.div_(self.world)

    def zero_grad(self) -> None:
        self.flat.zero_()

    def broadcast_parameters(self, src: int = 0) -> None:
        if self.world == 1:
            return
        with torch.no_grad():
            for t in list(self.model.parameters()) + [b for b in self.model.buffers() if b.dtype.is_floating_point or b.dtype == torch.int64]:
                dist.broadcast(t.data, src=src, group=self.group)
        inv = getattr(self.model, "invalidate", None)
        if callable(inv):
            inv()                               # packed weight arena follows the new values
