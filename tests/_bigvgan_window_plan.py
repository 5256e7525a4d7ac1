"""The window plan of fs2_bigvgan_window (csrc/bigvgan.cu, DESIGN.md section 18) restated in Python from the layer shapes:
the chain of tests/_ups_window_plan.py with BigVGAN's reaches.  An Activation1d reads ACT rows on each side (its 2x
upsampling reads 3 input rows around each 2x sample, its low-pass 6 2x samples around each output row), so an AMP block
reads its convolutions' reaches plus ACT per activation, and conv_post reads 3 rows of activation_post's output."""
import _ups_window_plan as P

ACT = 5
POST = P.CONV_REACH + ACT


def ceil32(c: int) -> int:
    return (c + 31) // 32 * 32


def block_reach(resblock: str, k: int, dil) -> int:
    """Rows an AMP block reads on each side, layer by layer: AMPBlock1 a1, c1 (dilation d), a2, c2 (dilation 1) per
    step; AMPBlock2 a, c (dilation d)."""
    half = (k - 1) // 2
    if str(resblock) == "1":
        return sum(ACT + half * d + ACT + half for d in dil[:3])
    return sum(ACT + half * d for d in dil[:2])


def stack_reach(cfg) -> int:
    return max(block_reach(cfg["resblock"], k, d) for k, d in zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"]))


def reaches(cfg):
    """{layer name: rows its input must hold on each side of a chunk}, from the audio back (names as in _ups_window_plan)."""
    R, rates = stack_reach(cfg), cfg["upsample_rates"]
    out = {"post": POST}
    need = POST
    for s in reversed(range(len(rates))):
        need += R
        out[f"stack{s + 1}"] = need
        left, right = P.convt_reach(need, rates[s]), P.convt_reach_right(need, rates[s])
        assert left == right
        out[f"ups{s}"] = need = left
    out["pre"] = need + P.CONV_REACH
    return out


def level_halo(cfg, s: int) -> int:
    r = reaches(cfg)
    return r["ups0"] + P.CONV_REACH if s == 0 else cfg["upsample_rates"][s - 1] * r[f"ups{s - 1}"]


def ups(cfg):
    out = [1]
    for u in cfg["upsample_rates"]:
        out.append(out[-1] * u)
    return out


def level_rows(cfg, s: int, n: int) -> int:
    return n * ups(cfg)[s] + 2 * level_halo(cfg, s)


def exact_margins(cfg):
    """[(level, rows wrong at a side that is not an utterance edge after the level's last layer, rows the next layer reads
    beyond its core window)]: level 0 is wrong in 3 rows, level s+1 enters wrong in u_s / 2 rows and its stack widens
    that by R."""
    U, R, r = len(cfg["upsample_rates"]), stack_reach(cfg), reaches(cfg)
    out = [(0, P.CONV_REACH, level_halo(cfg, 0) - r["ups0"])]
    for s in range(1, U + 1):
        nxt = r[f"ups{s}"] if s < U else POST
        out.append((s, cfg["upsample_rates"][s - 1] // 2 + R, level_halo(cfg, s) - nxt))
    return out


def n_windows(cfg) -> int:
    r, U = reaches(cfg), len(cfg["upsample_rates"])
    return U + 2 + sum(r[f"ups{s}"] != level_halo(cfg, s) for s in range(U))


def widths(cfg):
    c0 = cfg["upsample_initial_channel"]
    return [c0 // 2 ** s for s in range(len(cfg["upsample_rates"]) + 1)]


def workspace_bytes(cfg, B: int, n: int) -> int:
    """fs2_bigvgan_window_workspace_bytes: the window descriptors, then five buffers of the largest level buffer (rows x
    padded width over every level; conv_pre's operand, 80 wide, included)."""
    act = max([level_rows(cfg, 0, n) * P.N_MELS] + [level_rows(cfg, s, n) * ceil32(c) for s, c in enumerate(widths(cfg))])
    return P._carve([3 * n_windows(cfg) * B * 8] + [B * act * 4] * 5)


def whole_call_workspace_bytes(cfg, B: int, L: int) -> int:
    """fs2_bigvgan_workspace_bytes: the lengths, then five buffers of max_s up_s C'_s floats per frame of B * Lmax."""
    act = max(u * ceil32(c) for u, c in zip(ups(cfg), widths(cfg)))
    return P._carve([(len(cfg["upsample_rates"]) + 1) * B * 8] + [B * L * act * 4] * 5)
