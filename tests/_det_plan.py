"""Python restatement of the deterministic train mode's ordered sums (csrc/train.cu, csrc/train_det.cu, DESIGN.md §26): the
workspace each `_det` entry carves, and the longest sequential fp32 chain one output passes through, for the float64
gates of tests/test_gpu_train_deterministic.py (`max|err| / sum|terms| <= n_chain * 2^-24`, as in tests/_train_plan.py).

The geometry is tests/_train_plan.py's: every grid comes from the shapes and fixed constants.  Nothing here takes the
device's SM count."""
import _train_plan as P

U24 = P.U24
SC_ROWS, SC_GROUP = 256, 256        # rows per chunk of the counting sort, rows per group of one id's sum
SC_MAX_IDS = 8192


def _a256(n):
    return (n + 255) // 256 * 256


def carve(*sizes):
    """Bytes of a bump allocation of `sizes` (each carve starts on a 256-byte boundary; the last is not padded)."""
    off = 0
    for s in sizes:
        off = _a256(off) + s
    return off


def gy(rows):
    return P.colsum(rows, 1)["grid_y"]


def ctas(rows):
    return P.warp_rows(rows)[0]


def grid_for(n, block, cap):
    return max(1, min(-(-n // block), cap))


def colsum_bytes(rows, C):
    return 0 if rows == 0 else carve(4 * gy(rows) * C)


def conv_wgrad_bytes(B, L, N, K, taps):
    M = B * L
    if M == 0:
        return 0
    ch = P.wgrad(B, L, N, K, taps)["chunks"]
    parts = [4 * ch * taps * N * K] if ch > 1 else []
    return carve(*parts, 4 * gy(M) * N)


def layernorm_bytes(rows, C):
    if rows == 0:
        return 0
    c = ctas(rows)
    return carve(4 * c * C, 4 * c * C, 4 * gy(c) * C)


def batchnorm_bytes(rows, C):
    return carve(8 * P.bn(rows)["grid_y"] * 2 * C, 8 * 2 * C)


def _scatter(rows, C, n):
    ch = -(-rows // SC_ROWS)
    return [4 * n * ch, 4 * (n + 1), 4 * (n + 1), 4 * rows, 4 * (-(-rows // SC_GROUP) + n) * C]


def embed_bytes(B, T, C, n_sym):
    rows = B * T
    return 0 if rows == 0 else carve(4 * rows, 4 * gy(rows), *_scatter(rows, C, n_sym))


def onehot_bytes(rows, C, n_bins):
    return 0 if rows == 0 else carve(*_scatter(rows, C, n_bins), 4 * gy(rows) * C)


def rowdot_bytes(rows, C):
    if rows == 0:
        return 0
    c = ctas(rows)
    return carve(4 * c * C, 4 * c, 4 * gy(c) * C)


def loss_bytes(B, T, L, odim):
    g1, g2 = grid_for(L * odim // 4, 256, 32), grid_for(max(L, T), 256, 16)
    return carve(8 * 8, 8 * 2 * g1 * B, 8 * 3 * g2 * B)


# ---- chain lengths --------------------------------------------------------------------------------------------------------
def colsum_chain(rows):
    """a row-lane's rows, the 8 lanes of its block, the grid.y partials in order, the += ."""
    g = gy(rows)
    return -(-rows // (g * 8)) + 8 + g + 1


def wgrad_chain(B, L, N, K, taps):
    """one chunk's FMA chain, the chunks in order, the += (one chunk: the chain and the +=)."""
    p = P.wgrad(B, L, N, K, taps)
    return p["per"] + p["chunks"] + 1


def layernorm_chain(rows):
    """dgamma / dbeta: a warp's rows, the 8 warps in order, the CTA partials through the ordered column sum, and the 8
    roundings of a term (tests/_train_plan.layernorm_chain)."""
    _, _, rpw = P.warp_rows(rows)
    return rpw + 8 + colsum_chain(ctas(rows)) + 8


def rowdot_chain(rows):
    """dw and dbias: a warp's rows, the 8 warps in order, the CTA partials through the ordered column sum, the product."""
    _, _, rpw = P.warp_rows(rows)
    return rpw + 8 + colsum_chain(ctas(rows)) + 1


def scatter_chain(count):
    """one id's table row: its rows in groups of 256 (in order), the groups in order, the += ."""
    return min(count, SC_GROUP) + -(-count // SC_GROUP) + 1


def dalpha_chain(rows, C):
    """per row a warp sum of C / 32 products per lane over 5 shuffle levels, then the rows through the ordered column sum."""
    return -(-C // 32) + 5 + 1 + colsum_chain(rows)


# ---- kernel names ---------------------------------------------------------------------------------------------------------
# the default path's float-atomic kernels (demangled names up to the argument list) -- exactly these, and no others
DEFAULT_ATOMIC = {
    "colsum_kernel<false>", "wgrad_kernel<false>", "layernorm_backward_kernel<2, false>", "layernorm_backward_kernel<3, false>",
    "bn_stats_kernel<false>", "bn_backward_sums_kernel<false>", "bn_backward_apply_kernel<false>", "embed_backward_kernel<false>",
    "onehot_linear_backward_kernel", "rowdot_backward_kernel<false>", "loss_mel_kernel<false>", "loss_seq_kernel<false>",
}
# the kernels of the ordered entries (wgrad_reduce_kernel also serves fs2_conv_wgrad_tc)
ORDERED = {
    "colsum_kernel<true>", "wgrad_kernel<true>", "layernorm_backward_kernel<2, true>", "layernorm_backward_kernel<3, true>",
    "bn_stats_kernel<true>", "bn_backward_sums_kernel<true>", "bn_backward_apply_kernel<true>", "embed_backward_kernel<true>",
    "rowdot_backward_kernel<true>", "loss_mel_kernel<true>", "loss_seq_kernel<true>", "scatter_hist_kernel", "scatter_scan_kernel",
    "scatter_rank_kernel", "scatter_group_sum_kernel", "scatter_id_sum_kernel", "ordered_sum_f64_kernel", "wgrad_reduce_kernel",
}


def short_name(demangled):
    """`void fs2::(anonymous namespace)::colsum_kernel<true>(float const*, ...)` -> `colsum_kernel<true>`"""
    d = demangled.replace("(anonymous namespace)", "")
    head = d[:d.index("(")] if "(" in d else d
    return head.split("::")[-1]
