"""fs2_melgan_window's window plan (csrc/melgan.cu, DESIGN.md section 11) restated in Python: the rows each layer reads
around a chunk of audio, the rows per utterance of every window buffer, where a window buffer sits in its utterance, the
rows whose values equal the whole call's, and the workspace bytes.

Levels: 0 = the first conv's output (1 row per frame), s = 1..4 = ConvTranspose s-1's output, which its ResStack reads
and rewrites (8, 64, 128, 256 rows per frame).  The reaches are derived here from the layer shapes alone, so that the
tests can hold them against the float64 oracle's dependency cone."""
HOP = 256
UP = (1, 8, 64, 128, 256)
STRIDES = (8, 8, 2, 2)
CIN = (512, 256, 128, 64)
COUT = (256, 128, 64, 32)
DILATIONS = (1, 3, 9)
RES_REACH = sum(DILATIONS)          # a ResStack: three k = 3 convolutions at dilations 1, 3, 9
CONV_REACH = 3                      # the first and last convolutions, k = 7
N_WINDOWS = 9                       # window descriptors: levels 0..4, ConvTranspose 1..3's inputs, the audio


def _convt_reach(out_reach: int, s: int) -> int:
    """Input rows a ConvTranspose1d(k = 2s, stride s, padding s/2) reads left of a core for `out_reach` output rows left
    of s times that core: output row o = s t + r reads input rows t-1, t (r < s/2) or t, t+1 (r >= s/2)."""
    o = -out_reach
    t, r = o // s, o % s
    return -(t - 1 if r < s // 2 else t)


def _convt_reach_right(out_reach: int, s: int) -> int:
    o = out_reach - 1                  # the last output row right of the core, core end at 0
    t, r = o // s, o % s
    return (t + 1 if r >= s // 2 else t) + 1


def reaches():
    """The rows each layer's input must hold on each side of a chunk, at its own rate, from the last conv back to the
    first: {name: reach}.  Names: 'conv0' (mel frames), 'convt0'..'convt3', 'res0'..'res3' (ResStack inputs), 'post'."""
    out = {"post": CONV_REACH}
    need = CONV_REACH
    for s in reversed(range(4)):
        need += RES_REACH
        out[f"res{s}"] = need
        left, right = _convt_reach(need, STRIDES[s]), _convt_reach_right(need, STRIDES[s])
        assert left == right
        out[f"convt{s}"] = need = left
    out["conv0"] = need + CONV_REACH
    return out


def convt_reach(s: int) -> int:
    return reaches()[f"convt{s}"]


def level_halo(s: int) -> int:
    return convt_reach(0) if s == 0 else STRIDES[s - 1] * convt_reach(s - 1)


def level_rows(s: int, n: int) -> int:
    """Rows per utterance of level s's buffer for a window of n frames."""
    return n * UP[s] + 2 * level_halo(s)


def convt_rows(s: int, n: int) -> int:
    """Rows per utterance of ConvTranspose s's input window; level_rows(s + 1) = stride * convt_rows(s)."""
    return n * UP[s] + 2 * convt_reach(s)


def level_margin(s: int) -> int:
    """Rows at a window side that is not an utterance edge whose values differ from the whole call's, on entry to level
    s (ConvTranspose s-1's phases at the edge read a row outside its input window); each residual block adds its
    dilation."""
    return 0 if s == 0 else STRIDES[s - 1] // 2


def exact_margins():
    """(level, margin after its ResStack, rows the next layer reads beyond its core window): the plan is exact when the
    margin never reaches into what the next layer reads."""
    out = []
    for s in range(1, 5):
        out.append((s, level_margin(s) + RES_REACH, level_halo(s) - (convt_reach(s) if s < 4 else CONV_REACH)))
    return out


def core(start: int, n_frames: int, olens: int):
    """Core frames [c0, c1) of a window, or None when it is empty."""
    c0, c1 = start, min(start + n_frames, olens)
    return (c0, c1) if 0 <= c0 < c1 else None


def windows(start: int, n_frames: int, olens: int):
    """Global [lo, hi) rows of every buffer of one utterance's window: {'level0'..'level4', 'convt1'..'convt3', 'audio'}
    (empty dict for an empty window)."""
    c = core(start, n_frames, olens)
    if c is None:
        return {}
    c0, c1 = c
    out = {"level0": (max(c0 - convt_reach(0), 0), c1 + convt_reach(0))}
    for s in range(4):
        lo, hi = max(c0 * UP[s] - convt_reach(s), 0), c1 * UP[s] + convt_reach(s)
        if s > 0:
            out[f"convt{s}"] = (lo, hi)
        out[f"level{s + 1}"] = (lo * STRIDES[s], hi * STRIDES[s])
    out["audio"] = (c0 * HOP, c1 * HOP)
    return out


def _align(off: int) -> int:
    return (off + 255) & ~255


def workspace_bytes(B: int, n: int) -> int:
    """fs2_melgan_window_workspace_bytes: window descriptors, the largest operand and three activation buffers, each
    256-byte aligned, plus 256 bytes of slack for the base pointer's alignment."""
    op = max([level_rows(0, n) * 80 * 7] + [convt_rows(s, n) * 3 * CIN[s] for s in range(4)]
             + [level_rows(s + 1, n) * 3 * COUT[s] for s in range(4)])
    act = max([level_rows(0, n) * 512] + [level_rows(s + 1, n) * COUT[s] for s in range(4)])
    off = 0
    for size in (3 * N_WINDOWS * B * 8, B * op * 4, B * act * 4, B * act * 4, B * act * 4):
        off = _align(off) + size
    return off + 256


def whole_call_workspace_bytes(B: int, L: int) -> int:
    """fs2_melgan_workspace_bytes: 196,608 bytes per frame of B * (Lmax + 10), plus the lengths."""
    frames = B * (L + 10)
    off = 0
    for size in (5 * B * 8, frames * 3 * 256 * 32 * 4, frames * 256 * 32 * 4, frames * 256 * 32 * 4, frames * 256 * 32 * 4):
        off = _align(off) + size
    return off + 256


def window_flop_overhead(n: int) -> float:
    """FLOP of one window of n frames over its n frames' share of the whole call, from shapes before tile rounding."""
    def flop(rows_of_level, rows_of_convt):
        f = rows_of_level(0) * 2 * 80 * 7 * 512
        for s in range(4):
            f += rows_of_convt(s) * 2 * 3 * CIN[s] * STRIDES[s] * COUT[s]
            f += rows_of_level(s + 1) * 3 * (2 * 3 * COUT[s] ** 2 + 2 * 2 * COUT[s] ** 2)
        f += rows_of_level(4) * 2 * 7 * 32
        return f
    return flop(lambda s: level_rows(s, n), lambda s: convt_rows(s, n)) / flop(lambda s: n * UP[s], lambda s: n * UP[s]) - 1
