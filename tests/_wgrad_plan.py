"""Python restatement of the tensor-core weight-gradient kernel's work decomposition (csrc/wgrad_tc.cu, `wgrad_plan`):
output tiles, taps, splits of the (utterance, time) chunk range and the workspace layout.  The CPU tests check it against
the library's workspace formula and use it to show what the GPU cases reach."""
import math

BM, BN, BT = 128, 128, 32          # output tile rows (dy channels) x columns (x channels); time steps per chunk
PLAN_CTAS, MAX_SPLITS, MIN_CHUNKS = 132, 64, 4
H100_SMS = 132                     # H100 SXM

# (N, K, taps) of every ConvFn of train_forward at the default hp (configs/default.yaml: adim 256, ddim 384, units 1024,
# FFN kernel 9, predictors 256 x 3, Postnet 256 x 5 on 80 mels)
TRAIN_SHAPES = [
    (256, 256, 1),    # encoder q, k, v, out
    (1024, 256, 9),   # encoder w_1
    (256, 1024, 1),   # encoder w_2
    (256, 256, 3),    # duration / energy / pitch predictor convolutions
    (384, 256, 1),    # decoder input Linear
    (384, 384, 1),    # decoder q, k, v, out
    (1024, 384, 9),   # decoder w_1
    (384, 1024, 1),   # decoder w_2
    (80, 384, 1),     # feat_out
    (256, 80, 5),     # Postnet first conv
    (256, 256, 5),    # Postnet middle convs
    (80, 256, 5),     # Postnet last conv
]


def cdiv(a, b):
    return -(-a // b)


def plan(B, L, N, K, taps):
    cpu = cdiv(L, BT)
    Q = B * cpu
    tiles = cdiv(N, BM) * cdiv(K, BN) * taps
    smax = max(1, min(Q // MIN_CHUNKS, MAX_SPLITS))

    def eff(s):
        u = tiles * s
        return u / (math.ceil(u / PLAN_CTAS) * PLAN_CTAS)

    best, best_eff = 1, eff(1)
    for s in range(2, smax + 1):
        if eff(s) > best_eff + 0.05:
            best, best_eff = s, eff(s)
    P = ((taps - 1) // 2 + 3) // 4 * 4           # x^T copy r is shifted right by P + r steps
    phases = 4 if taps > 1 else 1
    return {"cpu": cpu, "Q": Q, "tiles": tiles, "splits": best, "units": tiles * best, "Lp": (L + 3) // 4 * 4,
            "P": P, "phases": phases, "Lx": (L + P + phases - 1 + 3) // 4 * 4, "bounds": [s * Q // best for s in range(best + 1)]}


def ws_bytes(B, L, N, K, taps):
    if B * L == 0:
        return 0
    p = plan(B, L, N, K, taps)
    a = lambda v: (v + 255) // 256 * 256
    return a(p["splits"] * taps * N * K * 4) + a(B * N * p["Lp"] * 4) + a(p["phases"] * B * K * p["Lx"] * 4)


def box_starts(L, taps):
    """Time coordinates of the x^T boxes of every (chunk, tap): each a non-negative multiple of 4, in copy r's extent."""
    p = plan(1, L, 128, 128, taps)
    out = []
    for j in range(taps):
        sh = j - (taps - 1) // 2 + p["P"]
        r = (-sh) % 4
        out += [(t0 + sh + r, r, L + p["P"] + r) for t0 in range(0, L, 32)]
    return out


def split_inside_utterance(B, L, N, K, taps):
    p = plan(B, L, N, K, taps)
    return any(c % p["cpu"] != 0 for c in p["bounds"][1:-1])


# GPU cases (B, L, N, K, taps): every train shape, plus lengths at the edges of the decomposition
KERNEL_CASES = [(3, 70, N, K, t) for (N, K, t) in TRAIN_SHAPES] + [
    (16, 200, 1024, 384, 9),   # 648 units: CTAs walk several units; split boundaries inside utterances
    (2, 150, 80, 384, 1),      # 3 units: one per CTA
    (5, 1, 256, 80, 5),        # L = 1
    (4, 3, 1024, 256, 9),      # L < pad
    (3, 45, 80, 256, 5),       # L % 4 != 0, L % 32 != 0, edge tiles in N
    (7, 33, 256, 80, 5),       # one step past a chunk; edge tiles in K
    (1, 517, 384, 1024, 1),    # a single utterance over many splits
]
