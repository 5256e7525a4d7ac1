"""Python restatement of the launch geometry of the fp32 train kernels (csrc/train.cu): the grid each entry point computes,
the work one thread, warp or chunk does, and the longest sequential fp32 chain a single output passes through.

The CPU tests check that the GPU cases of tests/test_gpu_train_ops.py reach every regime change of this geometry; the GPU
tests bound each kernel's error by `n_chain * 2^-24` relative to the sum of the absolute values of the terms (the
a-priori worst case of a sequential fp32 chain of that length), so a bad first run cannot set a loose gate.

Chain lengths count one rounding per sequential add (or FMA) on the longest path from the inputs to an output, plus one for
the `+=` onto the caller's starting value where the entry accumulates.  Sums taken in double (BatchNorm) count only the
fp32 roundings around them."""

SMS = 132                    # H100 SXM
U24 = 2.0 ** -24             # unit roundoff of fp32 (round to nearest)


def cdiv(a, b):
    return -(-a // b)


def warp_rows(rows):
    """layernorm_backward / rowdot_backward: grid = min(rows / 8 + 1, 528) CTAs of 8 warps; warp w walks rows
    w, w + 8 * grid, ...  Returns (ctas, rows per warp min, rows per warp max)."""
    ctas = min(rows // 8 + 1, SMS * 4)
    warps = ctas * 8
    return ctas, rows // warps, cdiv(rows, warps)


def layernorm_chain(rows, C):
    """dgamma / dbeta: a warp's rows in registers, 8 warps through shared atomics, one global atomic per CTA, += , and
    the 8 roundings of a term (xhat: subtract, rstd's add, sqrt and divide, multiply; the product with dy).
    dx: the row's three warp sums (C / 32 per lane, 5 shuffle levels) and the final combine."""
    ctas, _, rpw = warp_rows(rows)
    return {"dgamma": rpw + 8 + ctas + 1 + 8, "dx": 3 * (C // 32 + 5) + 8}


def rowdot_chain(rows, C):
    """dw: every row of a CTA through one shared atomic per column, then one global atomic per CTA, += ; dbias: a warp's
    rows in a register, then one global atomic per warp, += ; y: C / 32 per lane, 5 shuffle levels, the bias."""
    ctas, _, rpw = warp_rows(rows)
    return {"dw": 8 * rpw + ctas + 1, "dbias": rpw + 8 * ctas + 1, "y": cdiv(C, 32) + 6}


def colsum(rows, C):
    """grid (C / 32, min(rows / 512 + 1, 64)); each of the grid.y * 8 row-lanes walks rows with that stride, 8 row-lanes
    meet in shared memory, one global atomic per grid.y block, += ."""
    gy = min(rows // 512 + 1, 64)
    per = cdiv(rows, gy * 8)
    return {"grid_x": cdiv(C, 32), "grid_y": gy, "rows_per_lane": per, "chain": per + 8 + gy + 1}


def bn(rows):
    """bn_stats / bn_backward_sums: grid.y = min(rows / 256 + 1, 128).  The sums run in double; the fp32 chain is the
    rounding of the statistics and of the per-element expression around them (and the += of dgamma, dbeta)."""
    return {"grid_y": min(rows // 256 + 1, 128), "chain": 10}


WG_T = 64


def wgrad(B, L, N, K, taps):
    """fs2_conv_wgrad (fp32): 64 x 64 output tiles x taps; the B*L rows split into
    chunks = min(ceil(528 / tiles), ceil(M / 256)) ranges of `per` rows, combined with atomics."""
    M = B * L
    tiles = cdiv(N, WG_T) * cdiv(K, WG_T) * taps
    chunks = max(1, min(cdiv(SMS * 4, tiles), cdiv(M, 256)))
    per = cdiv(M, chunks)
    bounds = [c * per for c in range(1, chunks) if c * per < M]
    inside = any(b % L != 0 for b in bounds)
    return {"tiles": tiles, "chunks": chunks, "per": per, "boundary_inside_utterance": inside,
            "chain": per + chunks + 1, "fwd_chain": K * taps + 2, "dgrad_chain": N * taps + 2}


def softmax(L):
    """attn_softmax / attn_softmax_backward: one warp per row; lane l takes keys l, l + 32, ...  Idle lanes: lanes without
    a key in the last sweep.  Chain: a lane's keys, 5 shuffle levels, the exp / divide / subtract around them."""
    kpl = cdiv(L, 32)
    return {"keys_per_lane": kpl, "idle_lanes": 32 * kpl - L, "chain": kpl + 5 + 4}


def bgemm(M, N, K):
    """fs2_bgemm: 64 x 64 output tiles, K in steps of 16, one FMA chain over K per output, then alpha."""
    return {"tiles_m": cdiv(M, 64), "tiles_n": cdiv(N, 64), "k_steps": cdiv(K, 16),
            "tail_m": M % 64, "tail_n": N % 64, "tail_k": K % 16, "chain": K + 1}


def embed_chain(rows, C):
    """dalpha: C / 32 per lane, 5 shuffle levels, then one global atomic per warp (rows of them), += ."""
    return cdiv(C, 32) + 5 + rows + 1


# ---- the GPU cases ----------------------------------------------------------------------------------------------------------
C2_B, C2_T, C2_L = 64, 100, 800              # tools/bench_train.py c2: B = 64, T = 100 phonemes, L = 800 frames

LN_ROWS = [1, 7, 9, 4223, 4224, 4225, 6400, 51200]
LN_CS = [256, 384]
ROWDOT_ROWS = [4225, 51200]
COLSUM_ROWS = [1, 7, 8, 513, 32769, 51200]
COLSUM_CS = [1, 31, 33, 80, 256, 1024]
BN_ROWS = [2, 255, 256, 257, 32768, 51200]
BN_CS = [33, 80, 256]
SOFTMAX_LS = [1, 31, 32, 33, 64, 65, 800]


def SOFTMAX_LENS(L):
    """lens of the five utterances of a softmax case: empty, one, L - 1, L and past L"""
    return [0, 1, max(L - 1, 0), L, L + 5]


BGEMM_DIMS = [1, 15, 16, 17, 63, 64, 65, 333, 800]
# the six products AttentionFn issues (train.py): q.k^T, pd.v, pd^T.dO, dO.v^T, dS.k, dS^T.q
BGEMM_PATTERNS = ["q.kT", "pd.v", "pdT.dO", "dO.vT", "dS.k", "dST.q"]


def bgemm_cases():
    """(pattern, M, N, K, heads): three rotations of BGEMM_DIMS, so every size sits in every one of M, N and K three
    times, rather than the full product; patterns and heads 1-3 cycle."""
    D, out = BGEMM_DIMS, []
    for r in range(3):
        for i in range(len(D)):
            idx = len(out)
            out.append((BGEMM_PATTERNS[idx % 6], D[i], D[(i + 3 * r + 1) % 9], D[(i + 5 * r + 2) % 9], 1 + idx % 3))
    return out


# (B, L, N, K, taps) of the fp32 convolution cases: every train shape at (3, 70) and at the c2 scale the model runs it at
# (encoder and duration predictor: 64 x 100 rows; energy / pitch predictors, decoder and Postnet: 64 x 800)
_ENC = [(256, 256, 1), (1024, 256, 9), (256, 1024, 1), (256, 256, 3)]
_DEC = [(256, 256, 3), (384, 256, 1), (384, 384, 1), (1024, 384, 9), (384, 1024, 1), (80, 384, 1), (256, 80, 5),
        (256, 256, 5), (80, 256, 5)]


def conv_cases(train_shapes):
    small = [(3, 70, N, K, t) for (N, K, t) in train_shapes]
    c2 = [(C2_B, C2_T, N, K, t) for (N, K, t) in _ENC] + [(C2_B, C2_L, N, K, t) for (N, K, t) in _DEC]
    edges = [(3, L, 80, 256, t) for t in (5, 9) for L in (1, (t - 1) // 2, (t - 1) // 2 + 1)]
    two_chunks = [(3, 100, 80, 256, 5)]          # 300 rows: two chunks of 150, the boundary inside the second utterance
    return small + c2 + edges + two_chunks


# weight-gradient-only cases: N, K tails of 1 and 65 (the fp32 tap GEMM itself needs K % 16 == 0 and N % 4 == 0)
WGRAD_TAIL_CASES = [(3, 70, 1, 65, 3), (3, 70, 65, 1, 5), (2, 45, 65, 65, 9), (5, 33, 1, 1, 1)]
