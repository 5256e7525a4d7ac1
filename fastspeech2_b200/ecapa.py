"""Batched ECAPA-TDNN speaker embeddings on the library's kernels (DESIGN.md section 28; csrc/ecapa.cu).

`ECAPAEncoder.from_checkpoint("embedding_model.ckpt")(wavs, lens) -> [B, D]` runs SpeechBrain's `spkrec-ecapa-voxceleb`
encoder (Fbank(n_mels=80), sentence mean normalisation, ECAPA_TDNN) on 16 kHz audio.  Row b is the network applied to
wavs[b, :lens[b]] alone, bit-identical to a call with that utterance alone in every math mode; samples past lens[b] are
never read.  A call allocates nothing, never synchronises and reads one status word back.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._kernel_module import Handles, _take, check_status, query_bytes, read_checkpoint, workspace

SAMPLE_RATE = 16000
HOP = 160
DILATIONS = (1, 2, 3, 4, 1)          # SpeechBrain's default; dilations are not stored in a checkpoint
BN_EPS = 1e-5


def _tdnn(p: str) -> list:
    return [f"{p}.conv.conv.weight", f"{p}.conv.conv.bias", f"{p}.norm.norm.weight", f"{p}.norm.norm.bias",
            f"{p}.norm.norm.running_mean", f"{p}.norm.norm.running_var"]


def architecture(shapes: dict, dilations=DILATIONS) -> dict:
    """The constructor arguments implied by a state dict's shapes {key: shape}: n_mels, channels C, the number of
    SE-Res2Net blocks, the Res2Net scale, every kernel size, the SE and attention widths, the MFA width M, D and whether
    the ASP has global context.  Raises ValueError for a missing key or a shape the network cannot have."""
    def get(k):
        if k not in shapes:
            raise ValueError(f"missing key {k}")
        return tuple(shapes[k])
    C, n_mels, k0 = get("blocks.0.conv.conv.weight")
    nb = 0
    while f"blocks.{nb + 1}.tdnn1.conv.conv.weight" in shapes:
        nb += 1
    if nb < 1:
        raise ValueError("missing key blocks.1.tdnn1.conv.conv.weight")
    scale = 1
    while f"blocks.1.res2net_block.blocks.{scale - 1}.conv.conv.weight" in shapes:
        scale += 1
    ks = [k0] + [get(f"blocks.{i}.res2net_block.blocks.0.conv.conv.weight")[2] for i in range(1, nb + 1)]
    M, mfa_in, km = get("mfa.conv.conv.weight")
    A, ctx_in, _ = get("asp.tdnn.conv.conv.weight")
    se = get("blocks.1.se_block.conv1.conv.weight")[0]
    D = get("fc.conv.weight")[0]
    if ctx_in not in (M, 3 * M):
        raise ValueError(f"key asp.tdnn.conv.conv.weight has {ctx_in} input channels, expected {3 * M} (or {M})")
    if scale < 2 or C % (16 * scale):
        raise ValueError(f"channels C = {C} must be a multiple of 16 * res2net scale = {16 * scale}")
    if len(dilations) != nb + 2:
        raise ValueError(f"dilations must have {nb + 2} entries (got {len(dilations)})")
    return {"n_mels": n_mels, "channels": C, "n_blocks": nb, "scale": scale, "kernel_sizes": ks + [km], "dilations": list(dilations),
            "se_channels": se, "attention_channels": A, "mfa_channels": M, "lin_neurons": D, "global_context": ctx_in == 3 * M}


def expected_shapes(a: dict) -> dict:
    """{key: shape} of SpeechBrain's ECAPA_TDNN state dict for the architecture a (num_batches_tracked not listed)."""
    C, nm, M, A, se, D, sc = a["channels"], a["n_mels"], a["mfa_channels"], a["attention_channels"], a["se_channels"], a["lin_neurons"], a["scale"]
    out = {}

    def tdnn(p, cout, cin, k):
        out.update(dict(zip(_tdnn(p), [(cout, cin, k), (cout,), (cout,), (cout,), (cout,), (cout,)])))
    tdnn("blocks.0", C, nm, a["kernel_sizes"][0])
    for i in range(1, a["n_blocks"] + 1):
        tdnn(f"blocks.{i}.tdnn1", C, C, 1)
        for j in range(sc - 1):
            tdnn(f"blocks.{i}.res2net_block.blocks.{j}", C // sc, C // sc, a["kernel_sizes"][i])
        tdnn(f"blocks.{i}.tdnn2", C, C, 1)
        out.update({f"blocks.{i}.se_block.conv1.conv.weight": (se, C, 1), f"blocks.{i}.se_block.conv1.conv.bias": (se,),
                    f"blocks.{i}.se_block.conv2.conv.weight": (C, se, 1), f"blocks.{i}.se_block.conv2.conv.bias": (C,)})
    tdnn("mfa", M, a["n_blocks"] * C, a["kernel_sizes"][-1])
    tdnn("asp.tdnn", A, 3 * M if a["global_context"] else M, 1)
    out.update({"asp.conv.conv.weight": (M, A, 1), "asp.conv.conv.bias": (M,)})
    out.update({f"asp_bn.norm.{n}": (2 * M,) for n in ("weight", "bias", "running_mean", "running_var")})
    out.update({"fc.conv.weight": (D, 2 * M, 1), "fc.conv.bias": (D,)})
    return out


def _bn_affine(sd: dict, p: str):
    """A BatchNorm's eval affine (scale, shift) in float64, rounded once to fp32."""
    g, b, m, v = (sd[f"{p}.{n}"].double() for n in ("weight", "bias", "running_mean", "running_var"))
    s = g / torch.sqrt(v + BN_EPS)
    return [s.float(), (b - m * s).float()]


def ordered_tensors(sd: dict, a: dict) -> list:
    """The tensors fs2_ecapa_load takes, in its order (include/fs2_b200.h)."""
    t = []

    def tdnn(p):
        t.extend([sd[f"{p}.conv.conv.weight"], sd[f"{p}.conv.conv.bias"]] + _bn_affine(sd, f"{p}.norm.norm"))
    tdnn("blocks.0")
    for i in range(1, a["n_blocks"] + 1):
        tdnn(f"blocks.{i}.tdnn1")
        for j in range(a["scale"] - 1):
            tdnn(f"blocks.{i}.res2net_block.blocks.{j}")
        tdnn(f"blocks.{i}.tdnn2")
        t.extend(sd[f"blocks.{i}.se_block.conv{k}.conv.{n}"] for k in (1, 2) for n in ("weight", "bias"))
    tdnn("mfa")
    tdnn("asp.tdnn")
    t.extend([sd["asp.conv.conv.weight"], sd["asp.conv.conv.bias"]] + _bn_affine(sd, "asp_bn.norm"))
    t.extend([sd["fc.conv.weight"], sd["fc.conv.bias"]])
    return t


class ECAPAEncoder:
    """SpeechBrain's ECAPA-TDNN speaker encoder on the library's kernels.  math_mode: the convolutions' GEMMs ("fp32",
    "tf32", "3xf16" / "3xtf32", "f16"); the front end and every per-utterance reduction run in fp32 in all of them."""

    def __init__(self, state_dict: dict, math_mode: str = "3xf16", dilations=DILATIONS):
        if math_mode not in _lib.MATH_MODES:
            raise ValueError(f"math_mode must be one of {sorted(_lib.MATH_MODES)}")
        sd = {k: v for k, v in dict(state_dict).items() if not k.endswith("num_batches_tracked")}
        shapes = {k: tuple(v.shape) for k, v in sd.items() if torch.is_tensor(v)}
        self.arch = architecture(shapes, dilations)
        self.sd = _take(sd, list(expected_shapes(self.arch)), expected_shapes(self.arch))
        if sd:
            raise ValueError(f"unexpected key {sorted(sd)[0]}")
        a = self.arch
        if a["kernel_sizes"][-1] != 1:
            raise ValueError(f"the MFA's kernel size must be 1 (got {a['kernel_sizes'][-1]})")
        pad = max(d * (k - 1) // 2 for k, d in zip(a["kernel_sizes"][:-1], a["dilations"][:-1]))
        self.min_frames = pad + 1
        self.min_samples = pad * HOP      # 1 + N // 160 > pad
        self.math_mode = math_mode
        self.dim = a["lin_neurons"]
        self._handles = Handles("fs2_ecapa_destroy")
        self._ws = {}

    @classmethod
    def from_checkpoint(cls, path_or_dict, math_mode: str = "3xf16", dilations=DILATIONS) -> "ECAPAEncoder":
        """SpeechBrain's `embedding_model.ckpt` (a bare state dict), as a path or loaded."""
        return cls(read_checkpoint(path_or_dict, "state_dict", "an ECAPA_TDNN state dict"), math_mode, dilations)

    def __del__(self):
        if getattr(self, "_handles", None) is not None:
            self._handles.destroy_all()

    def config(self) -> _lib.ECAPAConfig:
        a = self.arch
        c = _lib.ECAPAConfig()
        for k in ("n_mels", "channels", "n_blocks", "scale", "se_channels", "attention_channels", "mfa_channels", "lin_neurons"):
            setattr(c, k, int(a[k]))
        c.global_context = int(a["global_context"])
        for i, (k, d) in enumerate(zip(a["kernel_sizes"], a["dilations"])):
            c.kernel_sizes[i], c.dilations[i] = int(k), int(d)
        return c

    def _create(self):
        h = C.c_void_p()
        _lib.check(_lib.load().fs2_ecapa_create(C.byref(h), _lib.MATH_MODES[self.math_mode], C.byref(self.config())), "fs2_ecapa_create")
        return h

    def _load(self, h, device) -> None:
        ts = [t.to(device).contiguous() for t in ordered_tensors(self.sd, self.arch)]
        arr = (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])
        _lib.check(_lib.load().fs2_ecapa_load(h, arr, len(ts), _lib.stream_ptr(device)), "fs2_ecapa_load")

    def _handle(self, device):
        return self._handles.get(device, 0, self._create, self._load)

    def _status_table(self):
        return [(_lib.FS2_ECAPA_BAD_LENGTH, f"every lens[b] must lie in [{self.min_samples}, Nmax] samples (at least "
                                            f"{self.min_frames} frames for the reflect padding)"),
                (_lib.FS2_ECAPA_RANGE, f"activations exceed the range of the fp16 operand planes in math_mode={self.math_mode!r} "
                                       f"(some GEMM input above {65504 / 16:g} in magnitude); use math_mode='fp32' or 'tf32'")]

    def check_size(self, B: int, N: int) -> None:
        """The limits of a call on B utterances of up to N samples, as ValueError."""
        rows = B * (1 + N // HOP)
        if rows >= 1 << 31:
            raise ValueError(f"B * (1 + Nmax // 160) = {rows} frame rows must stay below 2^31")
        if self.math_mode == "fp32" and rows > 65535 * 128:
            raise ValueError(f"math_mode='fp32' takes at most 65535 * 128 frame rows, B * (1 + Nmax // 160) = {rows}; split the batch")
        a = self.arch
        widest = max(a["kernel_sizes"][0] * a["n_mels"], a["n_blocks"] * a["channels"], a["mfa_channels"])
        if rows * widest >= 1 << 31:
            raise ValueError(f"B * (1 + Nmax // 160) * {widest} = {rows * widest} operand elements must stay below 2^31; split the batch")

    def _inputs(self, wavs, lens):
        if not torch.is_tensor(wavs) or wavs.dim() != 2 or wavs.shape[0] == 0 or wavs.shape[1] == 0:
            raise ValueError("wavs must be a non-empty [B, Nmax] tensor")
        if wavs.dtype != torch.float32:
            raise ValueError(f"wavs must be float32 (got {wavs.dtype})")
        if not torch.is_tensor(lens) or lens.dim() != 1 or lens.shape[0] != wavs.shape[0]:
            raise ValueError(f"lens must be a [B={wavs.shape[0]}] tensor")
        if lens.dtype.is_floating_point or lens.dtype == torch.bool or lens.is_complex():
            raise ValueError("lens must be an integer tensor")
        if not wavs.is_cuda:
            raise ValueError("wavs must be a CUDA tensor (the H100 path has no CPU fallback)")
        if lens.is_cuda and lens.device != wavs.device:
            raise ValueError("lens must be on the same device as wavs")
        if not lens.is_cuda and bool(((lens < self.min_samples) | (lens > wavs.shape[1])).any()):
            raise ValueError(self._status_table()[0][1])
        B, N = wavs.shape
        if N >= 1 << 31:
            raise ValueError("Nmax must stay below 2^31 samples")
        self.check_size(B, N)
        return wavs.contiguous(), lens.to(device=wavs.device, dtype=torch.int64).contiguous(), B, N

    def __call__(self, wavs: torch.Tensor, lens: torch.Tensor) -> torch.Tensor:
        """wavs [B, Nmax] fp32 at 16 kHz on the GPU, lens [B] samples (every lens[b] >= min_samples, 640 for SpeechBrain's
        model) -> embeddings [B, D] fp32."""
        wavs, lens, B, N = self._inputs(wavs, lens)
        dev = wavs.device
        h = self._handle(dev)
        ws = workspace(self._ws, dev, query_bytes("fs2_ecapa_workspace_bytes", h, B, N))
        emb = torch.empty((B, self.dim), dtype=torch.float32, device=dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.load().fs2_ecapa(h, _lib.ptr(wavs), _lib.ptr(lens), B, N, _lib.ptr(emb), _lib.ptr(status), _lib.ptr(ws),
                                             ws.numel(), _lib.stream_ptr(dev)), "fs2_ecapa")
        check_status(status, self._status_table())
        return emb

    def encode_batch(self, wavs: torch.Tensor, wav_lens=None, normalize: bool = False) -> torch.Tensor:
        """SpeechBrain's EncoderClassifier.encode_batch surface: wav_lens relative to Nmax (None: every row whole) become
        round(wav_lens * Nmax) samples; -> [B, 1, D], each row its own utterance's embedding as in __call__."""
        if normalize:
            raise ValueError("normalize=True (SpeechBrain's mean_var_norm_emb) is not supported")
        if torch.is_tensor(wavs) and wavs.dim() == 1:
            wavs = wavs[None]
        if not torch.is_tensor(wavs) or wavs.dim() != 2:
            raise ValueError("wavs must be a [B, Nmax] tensor")
        B, N = wavs.shape
        if wav_lens is None:
            lens = torch.full((B,), N, dtype=torch.int64)
        else:
            rel = torch.as_tensor(wav_lens, dtype=torch.float64).cpu()
            if rel.dim() != 1 or rel.shape[0] != B:
                raise ValueError(f"wav_lens must hold B={B} relative lengths")
            lens = torch.round(rel * N).to(torch.int64)
        return self(wavs, lens)[:, None, :]

    def stage(self, stage: int, x: torch.Tensor, lens: torch.Tensor, L: int, width_out: int, rows_out: int) -> torch.Tensor:
        """fs2_op_ecapa_stage (per-layer tests): x on the GPU, lens [B] int64 on the GPU; -> [rows_out, width_out]."""
        dev = x.device
        B = lens.shape[0]
        h = self._handle(dev)
        N = L if stage == 0 else (L - 1) * HOP
        ws = workspace(self._ws, dev, query_bytes("fs2_ecapa_workspace_bytes", h, B, N))
        out = torch.empty((rows_out, width_out), dtype=torch.float32, device=dev)
        status = torch.empty((1,), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.load().fs2_op_ecapa_stage(h, stage, _lib.ptr(x.contiguous()), _lib.ptr(lens), B, L, _lib.ptr(out), _lib.ptr(status),
                                                      _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev)), "fs2_op_ecapa_stage")
        check_status(status, self._status_table())
        return out
