"""The row kernels of csrc/rowwise.cu without a GPU: the restatements tests/test_gpu_row_kernels.py checks the kernels
against, the inputs it drives them with, and every argument the library must refuse before it launches anything.

* The duration rule clamp(round(exp(s) - 1), min=0).long() decides something only near the ties exp(s) = k + 1.5, where
  round-half-to-even and round-half-away differ for even k; random inputs almost never land there.  tie_set() builds
  the float32 values within +-64 ulps of fl32(log(k + 1.5)) for k <= 20,000 (and of -ln 2, the tie at -0.5), and the
  tests here assert that it holds the exact ties that tell the two rules apart.
* torch.bucketize (right=False) is a lower bound: the first i with !(bins[i] >= x), so NaN goes to n_edges.  edge_values()
  builds every edge, its float32 neighbours, +-0, +-inf, NaN and values past both ends; the tests assert that they reach
  every branch of the rule.
* The refusals run on a machine without a visible CUDA device only: a check that regressed would otherwise launch a
  kernel on a misaligned pointer.  Without a device a launch can only fail with FS2_ERR_CUDA, never FS2_ERR_INVALID.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib

F32 = np.float32
INT64_MAX = np.iinfo(np.int64).max
TIE_KMAX = 20000
TIE_SPAN = 64


# ---- the duration rule -------------------------------------------------------------------------------------------
def ulp32(v):
    """Spacing of float32 at |v| (float64 result)."""
    return np.spacing(np.abs(np.asarray(v, dtype=np.float64)).astype(F32)).astype(np.float64)


def step_f32(x, n):
    """x moved n float32 ulps (n may be negative, arrays broadcast): walks the ordered integer image of the bits."""
    x = np.asarray(x, dtype=F32)
    i = x.view(np.int32).astype(np.int64)
    ordered = np.where(i < 0, -(i & 0x7FFFFFFF), i) + np.asarray(n, dtype=np.int64)
    back = np.where(ordered < 0, (-ordered) | -0x80000000, ordered)
    return back.astype(np.int64).astype(np.int32).view(F32)


def tie_set(kmax=TIE_KMAX, span=TIE_SPAN):
    """float32 x within +-span ulps of fl32(log(k + 1.5)), k = 0..kmax, and of fl32(-ln 2)."""
    centres = np.log(np.arange(kmax + 1, dtype=np.float64) + 1.5).astype(F32)
    centres = np.append(centres, F32(-np.log(2.0)))
    x = step_f32(centres[:, None], np.arange(-span, span + 1)[None, :]).ravel()
    return np.unique(x)


def uniform_set(n=1_000_000, seed=0):
    return np.random.default_rng(seed).uniform(-10, 10, n).astype(F32)


def special_set():
    """+-0, +-inf, NaN, subnormals and the values past 43.67 where exp(x) - 1 exceeds the int64 range."""
    tiny = np.array([1e-45, 1e-40, 1.1754942e-38], dtype=F32)
    past = np.array([43.6, 43.66, 43.668, 43.67, 43.7, 44, 50, 88.7, 88.73, 89, 100, 1e30, 3.4e38], dtype=F32)
    return np.concatenate([np.array([0.0, -0.0, np.inf, -np.inf, np.nan], dtype=F32), tiny, -tiny, past,
                           step_f32(F32(43.668), np.arange(-32, 33))])


def tie_distance(x):
    """(k, d): the nearest tie exp(x) = k + 1.5 (k >= -1) in float64 and the distance to it in float32 ulps of k + 1.5."""
    e = np.exp(np.asarray(x, dtype=np.float64))
    k = np.floor(e - 1.0)              # e in [k + 1, k + 2): the tie inside is k + 1.5
    k = np.maximum(k, -1.0)
    d = np.abs(e - (k + 1.5)) / ulp32(k + 1.5)
    return k, d


def dur_truth(x):
    """clamp(round_half_even(exp(x) - 1), 0) in float64, saturated to int64 as the device's conversion does."""
    with np.errstate(over="ignore", invalid="ignore"):
        r = np.maximum(np.rint(np.exp(np.asarray(x, dtype=np.float64)) - 1.0), 0.0)
    out = np.where(r >= 2.0 ** 63, INT64_MAX, 0)
    ok = np.isfinite(r) & (r < 2.0 ** 63)
    out[ok] = r[ok].astype(np.int64)
    out[np.isposinf(r)] = INT64_MAX
    return out


def tie_half_even(k):
    """The duration at an exact tie exp(x) - 1 = k + 0.5 (k >= 0): the even one of k and k + 1."""
    return k + (k % 2)


def exact_ties(x, within=0.01):
    """Mask of x with exp(x) within `within` float32 ulps of a tie k + 1.5, k >= 0."""
    k, d = tie_distance(x)
    return (k >= 0) & (d < within) & (k < 2 ** 22)


def exact_tie_candidates(kmin, kmax, span=TIE_SPAN, within=0.01):
    """Only the x of the +-span-ulp windows around fl32(log(k + 1.5)), kmin <= k <= kmax, that are exact ties."""
    parts = []
    for lo in range(kmin, kmax + 1, 10000):
        centres = np.log(np.arange(lo, min(lo + 10000, kmax + 1), dtype=np.float64) + 1.5).astype(F32)
        x = step_f32(centres[:, None], np.arange(-span, span + 1)[None, :]).ravel()
        parts.append(x[exact_ties(x, within)])
    return np.unique(np.concatenate(parts))


# ---- bucket edges ------------------------------------------------------------------------------------------------
def bin_sets():
    """name -> float32 edges: the model's two variance_bins, duplicates with a 0 edge, and n_edges 1 and 3."""
    from fastspeech2_b200.weights import ModelDims, variance_bins
    e, p = variance_bins(ModelDims())
    return {
        "energy": e.numpy().astype(F32), "pitch": p.numpy().astype(F32),
        "dup_zero": np.array([-3, -1, -1, 0, 0, 0, 0.25, 2, 2, 2, 7], dtype=F32),
        "one": np.array([0.5], dtype=F32),
        "three": np.array([-1, 0, 1e-3], dtype=F32),
    }


def edge_values(bins):
    """Every edge, nextafter on either side, +-0, +-inf, NaN, and values below the first and above the last edge."""
    b = np.asarray(bins, dtype=F32)
    lo, hi = b.min(), b.max()
    extra = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, lo - 1, lo - abs(lo) - 1e6, hi + 1, hi + abs(hi) + 1e6,
                      -3.4e38, 3.4e38], dtype=F32)
    return np.concatenate([b, np.nextafter(b, F32(np.inf)), np.nextafter(b, F32(-np.inf)), extra]).astype(F32)


def bucket_branches(values, bins):
    """Which branch of the lower bound each value takes: below, equal an edge, between, above, NaN."""
    v, b = np.asarray(values, dtype=F32), np.asarray(bins, dtype=F32)
    out = np.full(v.shape, "between", dtype=object)
    out[np.isin(v, b)] = "equal"
    out[v < b.min()] = "below"
    out[v > b.max()] = "above"
    out[np.isnan(v)] = "nan"
    return out


# ---- restatements of the fused arithmetic (float32, one rounding per operation) ----------------------------------
def fused_rows(beta, rows, *, relu=False, alpha=None, pe=None, L=0, spk_table=None, spk=None, spk_L=0, head_c=None,
               head_b=None, head_scale=None, lens=None):
    """The row kernel with gamma = 0: LayerNorm gives beta exactly, then relu -> + (alpha * pe[row % L]) ->
    + spk_table[spk[row / spk_L]] -> head = fl32(y[head_c] + head_b) (a one-hot head_w) [* head_scale[row]] -> the
    rows past lens written as +0.  Returns (out [rows, C], head [rows] or None, padded mask)."""
    C = beta.shape[0]
    y = np.broadcast_to(np.asarray(beta, dtype=F32), (rows, C)).copy()
    r = np.arange(rows)
    if relu:
        y = np.maximum(y, F32(0))
    if pe is not None:
        y = (y + (F32(alpha) * pe[r % L]).astype(F32)).astype(F32)
    if spk_table is not None:
        ids = spk[r // spk_L]
        ok = (ids >= 0) & (ids < spk_table.shape[0])
        y[ok] = (y[ok] + spk_table[ids[ok]]).astype(F32)
    head = None
    if head_c is not None:
        head = (y[:, head_c] + F32(head_b)).astype(F32)
        if head_scale is not None:
            head = (head * head_scale).astype(F32)
    padded = np.zeros(rows, dtype=bool) if lens is None else (r % L) >= lens[r // L]
    y[padded] = 0
    if head is not None:
        head[padded] = 0
    return y, head, padded


def variance_rows(h, e_ids, p_ids, e_tab, e_bias, p_tab, p_bias):
    """(h + (p_tab[p] + p_bias)) + (e_tab[e] + e_bias): pitch first, each add rounded to float32."""
    pw = (p_tab[p_ids] + p_bias).astype(F32)
    ew = (e_tab[e_ids] + e_bias).astype(F32)
    return ((h + pw).astype(F32) + ew).astype(F32)


# ---- CPU tests of the plan -----------------------------------------------------------------------------------------
def test_step_f32_walks_ulps():
    x = np.array([1.0, -1.0, 0.0, -0.0, 1e-45], dtype=F32)
    assert np.array_equal(step_f32(x, 1), np.nextafter(x, F32(np.inf)))
    assert np.array_equal(step_f32(x, -1), np.nextafter(x, F32(-np.inf)))
    assert step_f32(F32(1.0), 2**23).item() == 2.0


def test_tie_set_separates_half_even_from_half_away():
    """At least 20 exact ties with even k: there rint and roundf disagree, so the set pins rintf."""
    x = tie_set()
    assert x.size > 1_900_000 and x.dtype == F32     # windows of neighbouring k overlap at large k
    m = exact_ties(x)
    k, _ = tie_distance(x[m])
    even = int(np.sum(k % 2 == 0))
    print(f"MEASURED tie_set exact_ties {int(m.sum())} even_k {even}")
    assert even >= 20
    # exp(x) correctly rounded to float32 is the tie itself, where half to even gives k and half away k + 1
    assert np.all(np.exp(x[m].astype(np.float64)).astype(F32) == (k + 1.5).astype(F32))
    assert np.all(tie_half_even(k) != k + 1) == (even == k.size) and np.sum(tie_half_even(k) == k) == even


def test_exact_tie_candidates_extend_the_tie_set():
    """The device test adds the exact ties of k in (20,000, 60,000]: a margin of even-k ties for where the device's expf
    is not correctly rounded."""
    x = exact_tie_candidates(TIE_KMAX + 1, 3 * TIE_KMAX)
    k, d = tie_distance(x)
    assert np.all(d < 0.01) and np.all(k > TIE_KMAX)
    print(f"MEASURED extra_exact_ties {x.size} even_k {int(np.sum(k % 2 == 0))}")
    assert np.sum(k % 2 == 0) >= 10


def test_tie_set_and_specials_reach_every_regime():
    x = np.concatenate([tie_set(), uniform_set(), special_set()])
    t = dur_truth(x)
    assert (t == 0).any() and (t == INT64_MAX).sum() >= 10 and (t > 10_000).any()
    assert np.isnan(x).any() and np.isposinf(x).any() and np.isneginf(x).any()
    assert (np.abs(x[np.isfinite(x)]) < 1.2e-38).sum() >= 6     # subnormals and the smallest normal
    k, d = tie_distance(x[np.isfinite(x) & (x < 17)])
    assert (d <= 2).sum() > 1000 and (d > 2).sum() > 1_000_000   # both sides of the 2-ulp line are populated
    assert np.isclose(np.exp(-np.log(2.0)), 0.5)


def test_edge_values_span_every_bucketize_branch():
    for name, b in bin_sets().items():
        v = edge_values(b)
        got = set(bucket_branches(v, b))
        want = {"below", "equal", "between", "above", "nan"} - (set() if np.unique(b).size > 1 else {"between"})
        assert got == want, (name, got)
        ids = torch.bucketize(torch.from_numpy(v), torch.from_numpy(b))
        assert int(ids[np.isnan(v)].min()) == b.size                          # NaN -> n_edges
        assert int(ids.min()) == 0 and int(ids.max()) == b.size
        eq = np.isin(v, b) & np.isfinite(v)
        first = np.searchsorted(b, v[eq], side="left")                           # lower bound at an edge
        assert np.array_equal(ids[torch.from_numpy(eq)].numpy(), first)
    assert {b.size for b in bin_sets().values()} >= {1, 3, 255}


def test_fused_rows_restatement():
    beta = np.array([-1.5, 0.25, 2.0, -0.0] * 64, dtype=F32)
    pe = np.arange(3 * 256, dtype=F32).reshape(3, 256) / 7
    out, head, pad = fused_rows(beta, 6, relu=True, alpha=F32(0.5), pe=pe, L=3, head_c=1, head_b=F32(0.125),
                                lens=np.array([3, 1]))
    assert out.dtype == F32 and out.shape == (6, 256)
    assert out[0, 0] == F32(0.5) * pe[0, 0]                                  # relu(-1.5) = 0
    assert np.array_equal(pad, [False, False, False, False, True, True])
    assert np.all(out[4:] == 0) and np.all(head[4:] == 0)
    assert head[2] == F32(F32(0.25) + F32(0.5) * pe[2, 1]) + F32(0.125)


# ---- refusals: FS2_ERR_INVALID with a message naming the field, before any launch --------------------------------
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="refusal tests run only where no CUDA device is visible")
A = 0x10000                  # fake, 256-byte aligned device addresses: never dereferenced on the host


def _refused(rc, *words):
    msg = _lib.load().fs2_last_error().decode()
    assert rc == -1, (rc, msg)
    for w in words:
        assert w in msg, (w, msg)


def _desc(**kw):
    base = dict(x=A, ldx=256, gamma=A + 0x1000, beta=A + 0x2000, eps=1e-5, rows=8, C=256, out=A + 0x3000, ldo=256)
    base.update(kw)
    return _lib.RowNormDesc(**base)


ROW_NORM_REFUSALS = [
    (dict(x=A + 4), "x must be 16-byte aligned"),
    (dict(resid=A + 0x4004, ldr=256), "resid must be 16-byte aligned"),
    (dict(out=A + 0x3008), "out must be 16-byte aligned"),
    (dict(gamma=A + 0x100C), "gamma must be 16-byte aligned"),
    (dict(beta=A + 0x2004), "beta must be 16-byte aligned"),
    (dict(pe=A + 0x5004, alpha=A + 0x6000, L=8), "pe must be 16-byte aligned"),
    (dict(head_w=A + 0x7004, head_b=A + 0x8000), "head_w must be 16-byte aligned"),
    (dict(spk_table=A + 0x9004, spk=A + 0xA000, n_spk=2, spk_L=4), "spk_table must be 16-byte aligned"),
    (dict(split_out=A + 0xB002), "split_out must be 8-byte aligned"),
    (dict(pe=A + 0x5000, alpha=A + 0x6000, L=0), "pe needs"),
    (dict(pe=A + 0x5000, L=8), "pe needs alpha"),
    (dict(head_out=A + 0xC000), "head_out"),
    (dict(dur_out=A + 0xC000), "dur_out"),
    (dict(head_scale=A + 0xC000, head_out=A + 0xD000), "head_scale"),
    (dict(head_w=A + 0x7000), "head_b"),
    (dict(C=128), "C=128"),
    (dict(C=512, ldx=512, ldo=512), "C=512"),
    (dict(x=0), "x is null"),
    (dict(gamma=0), "gamma"),
    (dict(beta=0), "beta"),
    (dict(ldx=258), "ldx"),
    (dict(resid=A + 0x4000, ldr=255), "ldr"),
    (dict(ldo=257), "ldo"),
    (dict(lens=A + 0xE000, L=0), "lens"),
    (dict(spk_table=A + 0x9000, n_spk=2, spk_L=4), "spk_table"),
    (dict(out=0), "no output"),
]


@no_device
@pytest.mark.parametrize("fields,words", ROW_NORM_REFUSALS, ids=[w for _, w in ROW_NORM_REFUSALS])
def test_row_norm_refuses(fields, words):
    d = _desc(**fields)
    _refused(_lib.load().fs2_op_row_norm(C.byref(d), None), words)


@no_device
def test_row_norm_refuses_a_null_descriptor():
    _refused(_lib.load().fs2_op_row_norm(None, None), "null descriptor")


@no_device
def test_layernorm_entry_refuses_misaligned_rows():
    lib = _lib.load()
    _refused(lib.fs2_op_layernorm(A + 4, None, A, A, 1e-5, 8, 256, A, None), "x must be 16-byte aligned")
    _refused(lib.fs2_op_layernorm(A, A + 8, A, A, 1e-5, 8, 256, A, None), "resid must be 16-byte aligned")
    _refused(lib.fs2_op_layernorm(A, None, A, A, 1e-5, 8, 320, A, None), "C=320")


def _embed(**kw):
    a = dict(xs=A, table=A + 0x1000, n_sym=10, pe=A + 0x2000, alpha=A + 0x3000, B=2, T=4, C=256, out=A + 0x4000, planes=None,
             lens=None)
    a.update(kw)
    return _lib.load().fs2_embed_posenc(*a.values(), None)


@no_device
@pytest.mark.parametrize("fields,words", [
    (dict(table=A + 0x1004), "table must be 16-byte aligned"),
    (dict(pe=A + 0x2008), "pe must be 16-byte aligned"),
    (dict(out=A + 0x400C), "out must be 16-byte aligned"),
    (dict(planes=A + 0x5002), "planes must be 8-byte aligned"),
    (dict(C=192), "C=192"),
    (dict(n_sym=0), "n_sym"),
    (dict(xs=None), "null"),
    (dict(alpha=None), "null"),
], ids=["table", "pe", "out", "planes", "C", "n_sym", "xs", "alpha"])
def test_embed_posenc_refuses(fields, words):
    _refused(_embed(**fields), words)


def _vea(**kw):
    a = dict(hm=A, e_val=A + 0x1000, p_val=A + 0x2000, e_bins=A + 0x3000, p_bins=A + 0x4000, n_edges=255, e_tab=A + 0x5000,
             e_bias=A + 0x6000, p_tab=A + 0x7000, p_bias=A + 0x8000, rows=16, C=256, out=A + 0x9000, planes=None, planes_lo=0,
             e_ids=None, p_ids=None, lens=None, L=0)
    a.update(kw)
    return _lib.load().fs2_op_variance_embed_add(*a.values(), None)


@no_device
@pytest.mark.parametrize("fields,words", [
    (dict(hm=A + 4), "hm must be 16-byte aligned"),
    (dict(e_tab=A + 0x5004), "e_tab must be 16-byte aligned"),
    (dict(e_bias=A + 0x6008), "e_bias must be 16-byte aligned"),
    (dict(p_tab=A + 0x700C), "p_tab must be 16-byte aligned"),
    (dict(p_bias=A + 0x8004), "p_bias must be 16-byte aligned"),
    (dict(out=A + 0x9004), "out must be 16-byte aligned"),
    (dict(planes=A + 0xA002), "planes must be 8-byte aligned"),
    (dict(lens=A + 0xB000, L=0), "lens needs L"),
    (dict(C=128), "C=128"),
    (dict(n_edges=-1), "n_edges"),
    (dict(hm=None), "null"),
    (dict(out=None), "null"),
], ids=["hm", "e_tab", "e_bias", "p_tab", "p_bias", "out", "planes", "lens", "C", "n_edges", "null_hm", "no_output"])
def test_variance_embed_add_refuses(fields, words):
    _refused(_vea(**fields), words)


@no_device
def test_one_hot_refuses():
    lib = _lib.load()
    _refused(lib.fs2_one_hot(A, 4, 256, A + 0x1004, None), "out must be 16-byte aligned")
    _refused(lib.fs2_one_hot(A, 4, 6, A + 0x1000, None), "n_bins")
    _refused(lib.fs2_one_hot(None, 4, 8, A, None), "null")
