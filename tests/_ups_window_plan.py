"""The window plan of an upsampling chain (csrc/vocoder_window.cuh, DESIGN.md section 11) restated in Python for
fs2_melgan_window (csrc/melgan.cu) and fs2_hifigan_window (csrc/hifigan.cu, DESIGN.md section 17): the rows each layer
reads around a chunk of audio, the rows per utterance of every window buffer, where a window buffer sits in its
utterance, the rows whose values equal the whole call's, and each vocoder's workspace bytes and FLOP overhead.

Levels: 0 = the first conv's output (1 row per frame), s = 1 .. U = upsampling s-1's output, which its residual stack
reads and rewrites (up_s rows per frame).  Layer names: 'pre' (the first conv's input, mel frames), 'ups{s}' (upsampling
s's input, level s), 'stack{s}' (level s's residual stack input), 'post' (the last conv's input).  The reaches are derived
here from the layer shapes alone, so that the tests can hold them against the float64 oracle's dependency cone."""
from dataclasses import dataclass

HOP = 256
N_MELS = 80
CONV_REACH = 3                      # the first and last convolutions, k = 7


@dataclass(frozen=True)
class Chain:
    vocoder: str                    # "melgan" or "hifigan": the buffer layout of the workspace
    rates: tuple                    # upsample rates u_s (ConvTranspose1d k = 2u, stride u, padding u / 2)
    widths: tuple                   # channels of levels 0 .. U
    R: int                          # rows a residual stack reads on each side
    margin0: int                    # rows of level 0 wrong at a window side that is not an utterance edge
    tail: int                       # frames each utterance runs past olens
    stack_taps: int                 # sum of taps x K / C over a residual stack's convolutions (its MACs per row / C^2)


def melgan():
    """seungwonpark/melgan: a ResStack is three blocks of a k = 3 conv at dilations 1, 3, 9 and a 1x1 conv with its 1x1
    shortcut; the first conv's producer reads mel frames for every tap; 10 tail frames."""
    return Chain("melgan", (8, 8, 2, 2), (512, 256, 128, 64, 32), R=1 + 3 + 9, margin0=0, tail=10, stack_taps=3 * (3 + 2))


def hifigan(cfg):
    """A hifi-gan config: R = the largest resblock's reach (ResBlock1 sum_m (k-1)/2 (d_m + 1), ResBlock2 sum_m (k-1)/2 d_m);
    conv_pre's native taps leave its 3 outer rows wrong; no tail."""
    one = str(cfg["resblock"]) == "1"
    steps, per = (3, 6) if one else (2, 2)
    R = max(sum((k - 1) // 2 * (d + one) for d in dil[:steps])
            for k, dil in zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"]))
    rates, c0 = tuple(cfg["upsample_rates"]), cfg["upsample_initial_channel"]
    return Chain("hifigan", rates, tuple(c0 // 2 ** s for s in range(len(rates) + 1)), R=R, margin0=CONV_REACH, tail=0,
                 stack_taps=sum(per * k for k in cfg["resblock_kernel_sizes"]))


def ups(c):
    """Cumulative upsampling of levels 0 .. U."""
    out = [1]
    for u in c.rates:
        out.append(out[-1] * u)
    return out


def convt_reach(out_reach: int, u: int) -> int:
    """Input rows a ConvTranspose1d(k = 2u, stride u, padding u/2) reads left of a core for `out_reach` output rows left
    of u times that core: output row o = u t + r reads input rows t-1, t (r < u/2) or t, t+1 (r >= u/2)."""
    t, r = divmod(-out_reach, u)
    return -(t - 1 if r < u // 2 else t)


def convt_reach_right(out_reach: int, u: int) -> int:
    t, r = divmod(out_reach - 1, u)      # the last output row right of the core, core end at 0
    return (t + 1 if r >= u // 2 else t) + 1


def reaches(c):
    """{layer name: rows its input must hold on each side of a chunk, at its own rate}, from the last conv back."""
    out = {"post": CONV_REACH}
    need = CONV_REACH
    for s in reversed(range(len(c.rates))):
        need += c.R
        out[f"stack{s + 1}"] = need
        left, right = convt_reach(need, c.rates[s]), convt_reach_right(need, c.rates[s])
        assert left == right
        out[f"ups{s}"] = need = left
    out["pre"] = need + CONV_REACH
    return out


def ups_reach(c, s: int) -> int:
    """r_s: upsampling s's input reach."""
    return reaches(c)[f"ups{s}"]


def level_halo(c, s: int) -> int:
    """h_s: rows of level s on each side of its core, h_0 = r_0 + margin0, h_{s+1} = u_s r_s."""
    return ups_reach(c, 0) + c.margin0 if s == 0 else c.rates[s - 1] * ups_reach(c, s - 1)


def level_rows(c, s: int, n: int) -> int:
    """Rows per utterance of level s's buffer for a window of n frames."""
    return n * ups(c)[s] + 2 * level_halo(c, s)


def ups_rows(c, s: int, n: int) -> int:
    """Rows per utterance of upsampling s's input window; level_rows(s + 1) = u_s * ups_rows(s)."""
    return n * ups(c)[s] + 2 * ups_reach(c, s)


def exact_margins(c):
    """[(level, rows wrong at a side that is not an utterance edge after the level's last layer, rows the next layer reads
    beyond its core window)]: the plan is exact when the first never exceeds the second.  Level 0 is wrong in margin0
    rows; level s+1 enters wrong in u_s / 2 rows (upsampling's edge phases read outside its operand) and its stack widens
    that by R."""
    U = len(c.rates)
    out = [(0, c.margin0, level_halo(c, 0) - ups_reach(c, 0))]
    for s in range(1, U + 1):
        nxt = ups_reach(c, s) if s < U else CONV_REACH
        out.append((s, c.rates[s - 1] // 2 + c.R, level_halo(c, s) - nxt))
    return out


def n_windows(c) -> int:
    """Window descriptors: levels 0 .. U, every upsampling input that is not its whole level's window, the audio."""
    return len(c.rates) + 2 + sum(ups_reach(c, s) != level_halo(c, s) for s in range(len(c.rates)))


def core(start: int, n_frames: int, olens: int):
    """Core frames [c0, c1) of a window, or None when it is empty."""
    c0, c1 = start, min(start + n_frames, olens)
    return (c0, c1) if 0 <= c0 < c1 else None


def windows(c, start: int, n_frames: int, olens: int):
    """Global [lo, hi) rows of every buffer of one utterance's window, clipped to its (olens + tail) * up_s rows:
    {'level0' .. 'levelU', 'ups0' .. 'ups{U-1}', 'audio'} (empty dict for an empty window)."""
    w = core(start, n_frames, olens)
    if w is None:
        return {}
    c0, c1 = w
    out = {}
    for s, up in enumerate(ups(c)):
        h, n = level_halo(c, s), (olens + c.tail) * up
        out[f"level{s}"] = (max(c0 * up - h, 0), min(c1 * up + h, n))
        if s < len(c.rates):
            r = ups_reach(c, s)
            out[f"ups{s}"] = (max(c0 * up - r, 0), min(c1 * up + r, n))
    out["audio"] = (c0 * HOP, c1 * HOP)
    return out


def _align(off: int) -> int:
    return (off + 255) & ~255


def _carve(sizes) -> int:
    """Bytes of buffers carved one after another, each 256-byte aligned, plus 256 bytes of slack for the base pointer's
    alignment."""
    off = 0
    for size in sizes:
        off = _align(off) + size
    return off + 256


def workspace_bytes(c, B: int, n: int) -> int:
    """fs2_<vocoder>_window_workspace_bytes: the window descriptors, then MelGAN's largest operand (rows x K over every
    producer) and three activation buffers (rows x C over every level), or HiFi-GAN's five buffers of the largest level
    buffer (conv_pre's operand, 80 wide, included)."""
    U, C = len(c.rates), c.widths
    desc = 3 * n_windows(c) * B * 8
    if c.vocoder == "melgan":
        op = max([level_rows(c, 0, n) * N_MELS * 7] + [ups_rows(c, s, n) * 3 * C[s] for s in range(U)]
                 + [level_rows(c, s + 1, n) * 3 * C[s + 1] for s in range(U)])
        act = max(level_rows(c, s, n) * C[s] for s in range(U + 1))
        return _carve([desc, B * op * 4] + [B * act * 4] * 3)
    act = max([level_rows(c, 0, n) * N_MELS] + [level_rows(c, s, n) * C[s] for s in range(U + 1)])
    return _carve([desc] + [B * act * 4] * 5)


def whole_call_workspace_bytes(c, B: int, L: int) -> int:
    """fs2_<vocoder>_workspace_bytes.  MelGAN: 196,608 bytes per frame of B * (Lmax + 10), plus the lengths.  HiFi-GAN:
    five buffers of max_s up_s C_s floats per frame of B * Lmax, plus the lengths."""
    U = len(c.rates)
    lens = (U + 1) * B * 8
    if c.vocoder == "melgan":
        frames = B * (L + c.tail)
        return _carve([lens, frames * 3 * 256 * 32 * 4] + [frames * 256 * 32 * 4] * 3)
    act = max(u * w for u, w in zip(ups(c), c.widths))
    return _carve([lens] + [B * L * act * 4] * 5)


def flop(c, level_rows_of, ups_rows_of) -> int:
    """FLOP of the generator's GEMMs and last conv over the given rows per level and per upsampling input, as the kernels
    run them (the upsamplings as 3-tap polyphase GEMMs)."""
    C, U = c.widths, len(c.rates)
    f = level_rows_of(0) * 2 * N_MELS * 7 * C[0]
    for s in range(U):
        f += ups_rows_of(s) * 2 * 3 * C[s] * c.rates[s] * C[s + 1]
        f += level_rows_of(s + 1) * 2 * c.stack_taps * C[s + 1] ** 2
    f += level_rows_of(U) * 2 * 7 * C[U]
    return f


def window_flop_overhead(c, n: int) -> float:
    """FLOP of one window of n frames over its n frames' share of the whole call, from shapes before tile rounding."""
    window = flop(c, lambda s: level_rows(c, s, n), lambda s: ups_rows(c, s, n))
    share = flop(c, lambda s: n * ups(c)[s], lambda s: n * ups(c)[s])
    return window / share - 1
