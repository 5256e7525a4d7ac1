"""fs2_hifigan_window's window plan (csrc/hifigan.cu, DESIGN.md section 17) restated from a hifi-gan config: the rows
each layer reads around a chunk of audio, the rows per utterance of every window buffer, where a window buffer sits in
its utterance, the rows whose values equal the whole call's, the workspace bytes and the FLOP overhead.

Levels: 0 = conv_pre's output (1 row per frame), s = 1 .. U = upsampling s-1's output, which its MRF reads and rewrites
(up_s rows per frame).  The reaches are derived here from the layer shapes alone, so that the tests can hold them against
the float64 oracle's dependency cone."""
HOP = 256
N_MELS = 80
CONV_REACH = 3                      # conv_pre and conv_post, k = 7


def rates(cfg):
    return list(cfg["upsample_rates"])


def ups(cfg):
    """Cumulative upsampling of levels 0 .. U."""
    out = [1]
    for u in rates(cfg):
        out.append(out[-1] * u)
    return out


def widths(cfg):
    c0 = cfg["upsample_initial_channel"]
    return [c0 // 2 ** s for s in range(len(rates(cfg)) + 1)]


def steps(cfg):
    return 3 if str(cfg["resblock"]) == "1" else 2


def resblock_reach(cfg, j):
    """Rows one resblock reads on each side: ResBlock1 sum_m (k-1)/2 (d_m + 1), ResBlock2 sum_m (k-1)/2 d_m."""
    k, dil = cfg["resblock_kernel_sizes"][j], cfg["resblock_dilation_sizes"][j][:steps(cfg)]
    return sum((k - 1) // 2 * (d + (1 if str(cfg["resblock"]) == "1" else 0)) for d in dil)


def mrf_reach(cfg):
    return max(resblock_reach(cfg, j) for j in range(len(cfg["resblock_kernel_sizes"])))


def convt_reach(out_reach: int, u: int) -> int:
    """Input rows a ConvTranspose1d(k = 2u, stride u, padding u/2) reads left of a core for `out_reach` output rows left
    of u times that core: output row o = u t + r reads input rows t-1, t (r < u/2) or t, t+1 (r >= u/2)."""
    t, r = divmod(-out_reach, u)
    return -(t - 1 if r < u // 2 else t)


def convt_reach_right(out_reach: int, u: int) -> int:
    t, r = divmod(out_reach - 1, u)      # the last output row right of the core, core end at 0
    return (t + 1 if r >= u // 2 else t) + 1


def reaches(cfg):
    """{name: rows each layer's input must hold on each side of a chunk, at its own rate}: 'conv_pre' (mel frames),
    'ups0' .. (the upsamplings' inputs), 'mrf1' .. 'mrfU' (the MRF inputs, level s), 'post'."""
    U, R = len(rates(cfg)), mrf_reach(cfg)
    out = {"post": CONV_REACH}
    need = CONV_REACH
    for s in reversed(range(U)):
        need += R
        out[f"mrf{s + 1}"] = need
        left, right = convt_reach(need, rates(cfg)[s]), convt_reach_right(need, rates(cfg)[s])
        assert left == right
        out[f"ups{s}"] = need = left
    out["conv_pre"] = need + CONV_REACH
    return out


def ups_reach(cfg, s: int) -> int:
    """r_s: upsampling s's input reach."""
    return reaches(cfg)[f"ups{s}"]


def level_halo(cfg, s: int) -> int:
    """h_s: rows of level s on each side of its core, h_0 = r_0 + 3, h_{s+1} = u_s r_s."""
    return ups_reach(cfg, 0) + CONV_REACH if s == 0 else rates(cfg)[s - 1] * ups_reach(cfg, s - 1)


def level_rows(cfg, s: int, n: int) -> int:
    """Rows per utterance of level s's buffer for a window of n frames."""
    return n * ups(cfg)[s] + 2 * level_halo(cfg, s)


def ups_rows(cfg, s: int, n: int) -> int:
    """Rows per utterance of upsampling s's input window; level_rows(s + 1) = u_s * ups_rows(s)."""
    return n * ups(cfg)[s] + 2 * ups_reach(cfg, s)


def exact_margins(cfg):
    """[(level, rows wrong at a side that is not an utterance edge after the level's last layer, rows the next layer reads
    beyond its core window)]: the plan is exact when the first never exceeds the second.  Level 0 is wrong in conv_pre's
    3 outer rows; level s+1 enters wrong in u_s / 2 rows (upsampling's edge phases read outside its operand) and its MRF
    widens that by R."""
    U, R = len(rates(cfg)), mrf_reach(cfg)
    out = [(0, CONV_REACH, level_halo(cfg, 0) - ups_reach(cfg, 0))]
    for s in range(1, U + 1):
        nxt = ups_reach(cfg, s) if s < U else CONV_REACH
        out.append((s, rates(cfg)[s - 1] // 2 + R, level_halo(cfg, s) - nxt))
    return out


def core(start: int, n_frames: int, olens: int):
    """Core frames [c0, c1) of a window, or None when it is empty."""
    c0, c1 = start, min(start + n_frames, olens)
    return (c0, c1) if 0 <= c0 < c1 else None


def windows(cfg, start: int, n_frames: int, olens: int):
    """Global [lo, hi) rows of every buffer of one utterance's window: {'level0' .. 'levelU', 'ups0' .. 'ups{U-1}',
    'audio'} (empty dict for an empty window)."""
    c = core(start, n_frames, olens)
    if c is None:
        return {}
    c0, c1 = c
    out = {}
    for s, up in enumerate(ups(cfg)):
        h = level_halo(cfg, s)
        out[f"level{s}"] = (max(c0 * up - h, 0), min(c1 * up + h, olens * up))
        if s < len(rates(cfg)):
            r = ups_reach(cfg, s)
            out[f"ups{s}"] = (max(c0 * up - r, 0), min(c1 * up + r, olens * up))
    out["audio"] = (c0 * HOP, c1 * HOP)
    return out


def _align(off: int) -> int:
    return (off + 255) & ~255


def workspace_bytes(cfg, B: int, n: int) -> int:
    """fs2_hifigan_window_workspace_bytes: 3 [B] descriptor rows per window buffer (U + 1 levels, U upsampling inputs,
    the audio), then five buffers of the largest level buffer per utterance, each 256-byte aligned, plus 256 bytes of slack
    for the base pointer's alignment."""
    U = len(rates(cfg))
    act = max([level_rows(cfg, 0, n) * N_MELS] + [level_rows(cfg, s, n) * c for s, c in enumerate(widths(cfg))])
    off = 0
    for size in [3 * (2 * U + 2) * B * 8] + [B * act * 4] * 5:
        off = _align(off) + size
    return off + 256


def whole_call_workspace_bytes(cfg, B: int, L: int) -> int:
    """fs2_hifigan_workspace_bytes: five buffers of max_s up_s C_s floats per frame of B * Lmax, plus the lengths."""
    U = len(rates(cfg))
    act = max(u * c for u, c in zip(ups(cfg), widths(cfg)))
    off = 0
    for size in [(U + 1) * B * 8] + [B * L * act * 4] * 5:
        off = _align(off) + size
    return off + 256


def flop(cfg, level_rows_of, ups_rows_of) -> int:
    """FLOP of the generator's GEMMs and conv_post over the given rows per level and per upsampling input, as the kernels
    run them (the upsamplings as 3-tap polyphase GEMMs)."""
    C, U = widths(cfg), len(rates(cfg))
    per = 6 if str(cfg["resblock"]) == "1" else 2
    f = level_rows_of(0) * 2 * N_MELS * 7 * C[0]
    for s in range(U):
        f += ups_rows_of(s) * 2 * 3 * C[s] * rates(cfg)[s] * C[s + 1]
        f += level_rows_of(s + 1) * sum(per * 2 * k * C[s + 1] ** 2 for k in cfg["resblock_kernel_sizes"])
    f += level_rows_of(U) * 2 * 7 * C[U]
    return f


def window_flop_overhead(cfg, n: int) -> float:
    """FLOP of one window of n frames over its n frames' share of the whole call, from shapes before tile rounding."""
    window = flop(cfg, lambda s: level_rows(cfg, s, n), lambda s: ups_rows(cfg, s, n))
    share = flop(cfg, lambda s: n * ups(cfg)[s], lambda s: n * ups(cfg)[s])
    return window / share - 1
