"""iSTFTNet's head restated per output sample in float64 numpy, independent of torch.istft: the formula
istftnet_head_kernel (csrc/istftnet.cu) implements.  test_istftnet_args.py holds it against the oracle's torch path."""
import numpy as np


def head(x, w, b, n_fft: int, hop: int):
    """x [T, C] (the last MRF's output), conv_post w [n_fft + 2, C, 7], b [n_fft + 2] -> audio [hop * T], float64.

    1. a = lrelu(x, 0.01); 2. padded row i is a[i - 1], row 0 is a[1] (0 when T < 2), rows outside [0, T] are 0;
    3. y[f, o] = b[o] + sum_{j, c} w[o, c, j] a_pad[f + j - 3] for frames f = 0 .. T;
    4. X_m = exp(y[f, m]) (cos + i sin)(sin(y[f, M + m])), M = n_fft / 2 + 1;
    5. frame f, sample k: (Re X_0 + (-1)^k Re X_{N/2} + 2 sum_{m=1}^{N/2-1} Re(X_m e^{2 pi i m k / N})) / N * w_hann[k];
       audio[n] = sum_f frame[f, p - hop f] / sum_f w_hann[p - hop f]^2 over frames f in [0, T] with 0 <= p - hop f < N,
       p = n + N / 2."""
    x, w, b = (np.asarray(v, dtype=np.float64) for v in (x, w, b))
    T, C = x.shape
    N, M = n_fft, n_fft // 2 + 1
    a = np.where(x > 0, x, 0.01 * x)
    # a_pad[i] for i = -3 .. T + 3, stored at i + 3
    pad = np.zeros((T + 7, C))
    pad[4: 4 + T] = a
    pad[3] = a[1] if T >= 2 else 0.0
    y = np.tile(b, (T + 1, 1))
    for j in range(7):
        y += pad[j: j + T + 1] @ w[:, :, j].T
    mag, ph = np.exp(y[:, :M]), np.sin(y[:, M:])
    re, im = mag * np.cos(ph), mag * np.sin(ph)
    k = np.arange(N)
    win = 0.5 - 0.5 * np.cos(2 * np.pi * k / N)
    frames = re[:, :1] + np.where(k % 2, -1.0, 1.0)[None] * re[:, N // 2: N // 2 + 1]
    for m in range(1, N // 2):
        th = 2 * np.pi * m * k / N
        frames = frames + 2 * (re[:, m: m + 1] * np.cos(th)[None] - im[:, m: m + 1] * np.sin(th)[None])
    frames = frames / N * win[None]
    p = np.arange(hop * T) + N // 2
    s, env = np.zeros(hop * T), np.zeros(hop * T)
    for d in range(N // hop + 1):
        f = p // hop - d
        kk = p - hop * f
        ok = (f >= 0) & (f <= T) & (kk < N)
        s[ok] += frames[f[ok], kk[ok]]
        env[ok] += win[kk[ok]] ** 2
    return s / env


def reach(n_fft: int, hop: int) -> int:
    """Last-level rows the head reads on each side of its samples' rows, derived from the index form: samples of row r
    are p in [hop r + N/2, hop (r + 1) + N/2), covered by frames [ceil((p - N + 1) / hop), floor(p / hop)], frame f reads
    rows f - 4 .. f + 2."""
    left = right = 0
    for r in range(64, 128):
        for p in range(hop * r + n_fft // 2, hop * (r + 1) + n_fft // 2):
            lo, hi = -(-(p - n_fft + 1) // hop), p // hop
            left, right = max(left, r - (lo - 4)), max(right, hi + 2 - r)
    return max(left, right)
