"""Host restatement of the fused optimizer's plan (csrc/optim.cu, DESIGN.md §15): the chunking of the parameter table, the
workspace it needs, and the per-step scalars the device computes in double (Noam rate, Adam step size, bias-correction
square root), written with the same operations in the same order so that the device values can be checked bit for bit.
numpy float64 arithmetic is IEEE round-to-nearest like the device's __dmul_rn / __dadd_rn; the exact product errors the
device takes from fma are formed here by Dekker's split, which gives the same exact value."""
import numpy as np

CHUNK = 65536            # elements per chunk (FS2_OPTIM_CHUNK)
BETA1, BETA2, EPS = 0.9, 0.98, 1e-9


def align256(n):
    return (n + 255) // 256 * 256


def chunks(numel):
    """Chunk count of each table entry and the first chunk of each (chunk c of entry t is [c - chunk0[t]] * CHUNK ...)."""
    counts = [(int(n) + CHUNK - 1) // CHUNK for n in numel]
    first, c = [], 0
    for k in counts:
        first.append(c)
        c += k
    return counts, first, c


def ws_bytes(numel):
    """Workspace of fs2_optim_*: fp64 sum of squares per chunk, the fp32 step size and bias-correction root per entry, then
    the reduction's scalars (norm as fp32, coefficient, skip flag: 16 bytes)."""
    n_chunks = chunks(numel)[2]
    return align256(8 * n_chunks) + align256(8 * len(numel)) + align256(16)


# ---- exact double-double helpers (the device uses fma for the product error) ---------------------------------------------
_SPLIT = 134217729.0     # 2^27 + 1


def _split(a):
    t = _SPLIT * a
    hi = t - (t - a)
    return hi, a - hi


def two_prod(a, b):
    """p = fl(a * b) and the exact error e = a * b - p (no overflow in the ranges used here)."""
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
    return p, e


def rsqrt(s):
    """Correctly rounded s ** -0.5 for s >= 1 (float64 arrays): 1 / sqrt(s), then one Newton correction from the exact
    residual 1 - s r^2 (a midpoint is never hit: s^-1/2 is not a 54-bit binary fraction for integer s)."""
    s = np.asarray(s, dtype=np.float64)
    r = 1.0 / np.sqrt(s)
    p, pe = two_prod(r, r)
    a, ae = two_prod(s, p)
    e = ((1.0 - a) - ae) - s * pe
    return r + (r * 0.5) * e


def pow_int(beta, n):
    """beta ** n for integer n >= 1 (int64 array) by squaring in double-double, rounded to double."""
    n = np.asarray(n, dtype=np.int64)
    rh, rl = np.ones(n.shape), np.zeros(n.shape)
    bh, bl = np.full(n.shape, beta), np.zeros(n.shape)
    k = n.copy()
    while np.any(k > 0):
        odd = (k & 1) == 1
        mh, ml = _dd_mul(rh, rl, bh, bl)
        rh, rl = np.where(odd, mh, rh), np.where(odd, ml, rl)
        bh, bl = _dd_mul(bh, bl, bh, bl)
        k >>= 1
    return rh + rl


def _dd_mul(ah, al, bh, bl):
    p, e = two_prod(ah, bh)
    e = e + (ah * bl + al * bh)
    hi = p + e
    return hi, e - (hi - p)


def noam_constants(model_size, factor, warmup):
    """The two host constants, grouped as NoamOpt.rate groups them: factor * model_size ** -0.5 and warmup ** -1.5."""
    return factor * model_size ** (-0.5), warmup ** (-1.5)


def noam_rate(step, model_size, factor, warmup):
    """lr of step (int64 array) as the device forms it: A * min(step ** -0.5, step * W) in double."""
    a, w = noam_constants(model_size, factor, warmup)
    s = np.asarray(step, dtype=np.float64)
    r = rsqrt(s)
    sw = s * w
    return a * np.where(sw < r, sw, r)


def adam_scalars(step, lr):
    """fp32 step size -lr / (1 - beta1 ** step) and fp32 sqrt(1 - beta2 ** step), as torch's Adam passes them."""
    step = np.asarray(step, dtype=np.int64)
    bc1 = 1.0 - pow_int(BETA1, step)
    bc2 = 1.0 - pow_int(BETA2, step)
    return (-(np.asarray(lr, dtype=np.float64) / bc1)).astype(np.float32), np.sqrt(bc2).astype(np.float32)
