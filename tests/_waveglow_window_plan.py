"""fs2_waveglow_window's window plan (csrc/waveglow.cu, DESIGN.md section 12) restated in Python from the layer shapes
alone: how far each flow reaches in step rows, the halo H, the mel frames and z steps a window reads, where a window's
buffer sits in its utterance, the rows whose values equal the whole call's after each flow and layer, and the workspace
bytes.  The tests hold the reaches against the float64 oracle's dependency cone.

A step row is 8 samples (n_group); a mel frame is 32 step rows."""
HOP, N_GROUP, N_MELS = 256, 8, 80
STEPS = HOP // N_GROUP                       # 32 step rows per frame
N_FLOWS, N_LAYERS, KERNEL = 12, 8, 3
DILATIONS = [2 ** i for i in range(N_LAYERS)]
UP_KERNEL, UP_STRIDE = 1024, 256             # ConvTranspose1d(80, 80, 1024, stride 256)
N_DESC = 6                                   # window descriptors per utterance (kWinRows)


def layer_reach(i: int) -> int:
    """Step rows WN layer i's in-layer convolution reads on each side: (k - 1) / 2 taps at dilation 2^i."""
    return (KERNEL - 1) // 2 * DILATIONS[i]


def flow_reach() -> int:
    """Step rows one flow reaches on each side: its 8 layers in sequence (start, end, coupling, 1x1 inverse and the
    early-noise concatenation are pointwise)."""
    return sum(layer_reach(i) for i in range(N_LAYERS))


def total_reach() -> int:
    """Step rows the 12 flows reach on each side of an output step: 3060."""
    return N_FLOWS * flow_reach()


def cond_reach() -> int:
    """Step rows a cond row reaches on each side: 3059.  Cond enters every WN layer after its in-layer convolution, so the
    first flow spreads it by layers 1 .. 7 only (254 rows) and each later flow by 255 through its state; the z path's
    3060 bounds it, which is what the halo covers."""
    return total_reach() - layer_reach(0)


def halo() -> int:
    """H: whole frames on each side of a window's core that cover the total reach."""
    return -(-total_reach() // STEPS)


def cond_mel_reach():
    """(left, right) mel frames cond frame f reads: the transposed convolution's 1024-sample kernel at stride 256 spans
    4 frames, so f reads f - 3 .. f."""
    return UP_KERNEL // UP_STRIDE - 1, 0


def mel_reach():
    """(left, right) mel frames a window reads around its core [s, s + n): [s - 99, s + n + 96)."""
    lo, hi = cond_mel_reach()
    return halo() + lo, halo() + hi


def buffer(start: int, n_frames: int, olens: int):
    """(f0, f1, c0, c1): the buffer's global frames [f0, f1) and the core [c0, c1), or None for an empty window."""
    c0, c1 = start, min(start + n_frames, olens)
    if not 0 <= c0 < c1:
        return None
    return max(0, c0 - halo()), min(olens, c1 + halo()), c0, c1


def buffer_frames(n_frames: int) -> int:
    """Frames per utterance of every window buffer: n + 2H, whatever the window's place."""
    return n_frames + 2 * halo()


def exact_margin(flows_done: int, layer: int | None = None, stage: str = "out") -> int:
    """Rows at a window side that is not an utterance edge whose values may differ from the whole call's.

    flows_done = j flows processed (in processing order k = 11 .. 0): the state and the WN start are exact at 255 j.
    Inside flow j, layer i: stage 'in' (the layer's input x) at 255 j + 2^i - 1, 'out' (its in-layer output, gate output
    and next x) at 255 j + 2^(i + 1) - 1."""
    base = flows_done * flow_reach()
    if layer is None:
        return base
    done = sum(layer_reach(l) for l in range(layer + (stage == "out")))
    return base + done


def plan_is_exact() -> bool:
    """The core of every window is exact after all 12 flows: the final margin fits inside the halo."""
    return exact_margin(N_FLOWS) <= halo() * STEPS


def _align(off: int) -> int:
    return (off + 255) & ~255


def _buffers(C: int, frames: int, planes: bool):
    """Byte sizes of plan()'s buffers after the lengths, in carving order."""
    rows = frames * STEPS
    out = [frames * 320 * 4, rows * 8 * 4, rows * C * 4, rows * C * 4]
    if planes:
        out.append(rows * C * 4)
    out += [rows * 2 * C * 4, rows * 2 * C * 4, rows * C * 4, rows * C * 4, rows * C * 4]
    if planes:
        out.append(rows * 640 * 4)
    if not (planes and 2 * C >= 640):
        out.append(rows * 640 * 4)
    return out


def _carve(sizes) -> int:
    off = 0
    for size in sizes:
        off = _align(off) + size
    return off + 256


def workspace_bytes(C: int, planes: bool, B: int, n_frames: int) -> int:
    """fs2_waveglow_window_workspace_bytes: the window descriptors, then the whole call's buffers for B utterances of
    n + 2H frames, each 256-byte aligned, plus 256 bytes of slack for the base pointer's alignment."""
    return _carve([N_DESC * B * 8] + _buffers(C, B * buffer_frames(n_frames), planes))


def whole_call_workspace_bytes(C: int, planes: bool, B: int, L: int) -> int:
    """fs2_waveglow_workspace_bytes: the two length vectors and the buffers for B utterances of Lmax frames."""
    return _carve([B * 8, B * 8] + _buffers(C, B * L, planes))


def window_flop_overhead(n_frames: int, sides: int = 2) -> float:
    """FLOP of a window over its core's share of the whole call, from shapes before tile rounding: every GEMM is linear
    in rows, so it is the buffer's frames over the core's, minus 1 (sides: halos present, 0, 1 or 2)."""
    return (n_frames + sides * halo()) / n_frames - 1
