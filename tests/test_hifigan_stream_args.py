"""Windowed HiFi-GAN without a GPU: the window plan (tests/_ups_window_plan.py) against the documented numbers and the
float64 oracle's NaN cone, its exactness over a grid of accepted configs and MelGAN's chain, the window workspace against
fs2_hifigan_window_workspace_bytes, argument validation of the C entry point and of `HiFiGANVocoder.window / stream /
forward(chunk_frames=)`, and the GPU case table's coverage."""
import ctypes as C
import itertools
import math
import os

import pytest
import torch

import _ups_window_plan as P
from conftest import REPO
from fastspeech2_b200 import _lib
from fastspeech2_b200.hifigan import CONFIGS, HiFiGANVocoder, check_config, load_config
from oracle import hifigan_oracle as O


# ---- the plan's numbers (DESIGN.md section 17) ---------------------------------------------------------------------------
def test_plan_numbers_for_v1_and_v3():
    v1, v3 = P.hifigan(CONFIGS["v1"]), P.hifigan(CONFIGS["v3"])
    assert v1.R == 60 and v3.R == 45
    assert [P.ups_reach(v1, s) for s in range(4)] == [10, 14, 47, 32]
    assert [P.ups_reach(v3, s) for s in range(3)] == [8, 8, 13]
    assert [P.level_halo(v1, s) for s in range(5)] == [13, 80, 112, 94, 64]
    assert [P.level_halo(v3, s) for s in range(4)] == [11, 64, 64, 52]
    assert P.reaches(v1)["pre"] == 13 and P.reaches(v3)["pre"] == 11
    assert [round(100 * P.window_flop_overhead(v1, n), 1) for n in (16, 32, 64, 128)] == [40.0, 20.0, 10.0, 5.0]
    assert [round(100 * P.window_flop_overhead(v3, n), 1) for n in (16, 32, 64, 128)] == [26.6, 13.3, 6.7, 3.3]
    assert round(P.workspace_bytes(v1, 64, 32) / 1e6) == 372 and round(P.workspace_bytes(v3, 64, 32) / 1e6) == 340
    for cfg in (v1, v3):
        assert round(P.whole_call_workspace_bytes(cfg, 64, 931) / 1e9, 2) == 9.76
        assert P.whole_call_workspace_bytes(cfg, 4, 2000) - P.whole_call_workspace_bytes(cfg, 4, 1000) == 163840 * 4000


@pytest.mark.parametrize("name", ["v1", "v3"])
def test_vocoder_plan_and_window_rows_match_the_restated_plan(name):
    cfg = P.hifigan(CONFIGS[name])
    v = HiFiGANVocoder(name)
    U = len(cfg.rates)
    assert v.window_plan() == {"reach": [P.ups_reach(cfg, s) for s in range(U)], "halo": [P.level_halo(cfg, s) for s in range(U + 1)],
                               "R": cfg.R}
    for B, n in ((1, 1), (7, 13), (64, 32)):
        assert v._window_rows(B, n)[0] == B * max(P.level_rows(cfg, s, n) for s in range(U + 1))
    assert v._window_rows(1, 32)[1] == f"B * (256 * n_frames + {2 * P.level_halo(cfg, U)})"


# ---- the reach: the plan against the float64 oracle's NaN cone -------------------------------------------------------
def _narrow(name, c0):
    return dict(load_config(name), upsample_initial_channel=c0)


# V1 and V3 topologies at reduced widths, and a resblock-2 config with other rates
CONE_CONFIGS = {
    "v1": _narrow("v1", 32),
    "v3": _narrow("v3", 32),
    "r2": {"resblock": "2", "upsample_rates": [4, 2, 8, 4], "upsample_kernel_sizes": [8, 4, 16, 8], "upsample_initial_channel": 32,
           "resblock_kernel_sizes": [5, 9], "resblock_dilation_sizes": [[1, 4], [3, 2]]},
}
ONE_FRAME_CONE = {"v1": 3258, "v3": 2582}          # samples a NaN mel frame reaches beyond its own 256


def _generator(cfg, seed=0):
    torch.manual_seed(seed)
    return O.Generator(cfg).double().eval()


@pytest.mark.parametrize("name", list(CONE_CONFIGS))
def test_plan_reach_matches_the_nan_cone(name):
    """A NaN mel frame just outside [c0 - h_0, c1 + h_0) leaves the chunk's audio finite; one just inside reaches it."""
    cfg = CONE_CONFIGS[name]
    gen = _generator(cfg)
    h0 = P.level_halo(P.hifigan(cfg), 0)
    c0, c1 = h0 + 3, h0 + 7
    frames = c1 + h0 + 3
    base = torch.randn(1, 80, frames, generator=torch.Generator().manual_seed(3), dtype=torch.float64) * 2 - 6
    for f, inside in ((c0 - h0 - 1, False), (c0 - h0, True), (c1 + h0 - 1, True), (c1 + h0, False)):
        mel = base.clone()
        mel[0, :, f] = float("nan")
        with torch.no_grad():
            audio = gen(mel)[0, 0, c0 * 256: c1 * 256]
        assert bool(torch.isnan(audio).any()) == inside, (name, f)
    if name in ONE_FRAME_CONE:
        f = h0 + 5
        mel = base.clone()
        mel[0, :, f] = float("nan")
        with torch.no_grad():
            nan = torch.isnan(gen(mel)[0, 0]).nonzero().flatten()
        r = ONE_FRAME_CONE[name]
        assert (int(nan.min()), int(nan.max()) + 1) == (f * 256 - r, (f + 1) * 256 + r), name


# ---- exactness over a grid of accepted configs --------------------------------------------------------------------------
def _rate_lists():
    """Orders of even factors of 256 into 1 .. 4 upsamplings."""
    out = set()
    for k in range(1, 5):
        for rs in itertools.product([2, 4, 8, 16, 32, 64, 128, 256], repeat=k):
            if math.prod(rs) == 256:
                out.add(rs)
    return sorted(out)


def _grid():
    """Accepted hifi-gan configs as chains, and MelGAN's chain."""
    yield P.melgan()
    for rates in _rate_lists():
        for resblock, kers, dils in (("1", [3, 7, 11], [[1, 3, 5]] * 3), ("2", [3, 5, 7], [[1, 2], [2, 6], [3, 12]]),
                                     ("1", [1], [[1, 1, 1]]), ("2", [31, 3], [[1024, 7], [1, 1]]), ("1", [5], [[2, 9, 1]])):
            cfg = {"resblock": resblock, "upsample_rates": list(rates), "upsample_kernel_sizes": [2 * u for u in rates],
                   "upsample_initial_channel": 32 << len(rates), "resblock_kernel_sizes": kers, "resblock_dilation_sizes": dils}
            check_config(load_config(cfg))
            yield P.hifigan(cfg)


def test_plan_is_exact_for_every_accepted_config_of_a_grid():
    n = 0
    for cfg in _grid():
        for level, wrong, room in P.exact_margins(cfg):
            assert wrong <= room, (cfg, level)
        for s, u in enumerate(cfg.rates):
            need = P.reaches(cfg)[f"stack{s + 1}"]
            assert u * P.ups_reach(cfg, s) >= need + u // 2, (cfg, s)
            assert P.ups_reach(cfg, s) <= P.level_halo(cfg, s), (cfg, s)    # the upsampling's operand fits in its level
        # every buffer of a window lies inside its level's rows, and each upsampling's input window inside its level's
        for start, nf, olens in ((0, 1, 1), (3, 5, 40), (17, 32, 900), (880, 32, 900)):
            w = P.windows(cfg, start, nf, olens)
            for s in range(len(cfg.rates) + 1):
                lo, hi = w[f"level{s}"]
                assert hi - lo <= P.level_rows(cfg, s, nf)
                if s < len(cfg.rates):
                    ulo, uhi = w[f"ups{s}"]
                    assert lo <= ulo and uhi <= hi and uhi - ulo <= P.ups_rows(cfg, s, nf)
                    assert w[f"level{s + 1}"] == (ulo * cfg.rates[s], uhi * cfg.rates[s])
        n += 1
    assert n >= 100


# ---- the workspace --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def handles():
    lib = _lib.load()
    hs = {}
    for name in ("v1", "v3"):
        for mode in (_lib.MATH_FP32, _lib.MATH_3XTF32):
            h = C.c_void_p()
            cfg = HiFiGANVocoder(name)._c_config()
            _lib.check(lib.fs2_hifigan_create(C.byref(h), mode, C.byref(cfg)), "fs2_hifigan_create")
            hs[name, mode] = h.value
    yield hs
    for h in hs.values():
        lib.fs2_hifigan_destroy(h)


def _ws(lib, h, B, n):
    out = C.c_size_t()
    rc = lib.fs2_hifigan_window_workspace_bytes(h, B, n, C.byref(out))
    return rc, out.value


@pytest.mark.gpu          # fs2_hifigan_create needs a device; the checks themselves run on the host
@pytest.mark.parametrize("name", ["v1", "v3"])
def test_window_workspace_is_the_plan_and_smaller_than_the_whole_call(handles, name):
    lib = _lib.load()
    h = handles[name, _lib.MATH_3XTF32]
    cfg = P.hifigan(CONFIGS[name])
    for B, n in ((1, 1), (1, 32), (7, 13), (64, 16), (64, 32), (64, 64), (3, 901)):
        rc, got = _ws(lib, h, B, n)
        assert rc == 0 and got == P.workspace_bytes(cfg, B, n), (B, n)
        for L in (n + 1, 2 * n, 931):                 # the whole call's grows with Lmax; a window's depends on n only
            if n < L:
                whole = C.c_size_t()
                assert lib.fs2_hifigan_workspace_bytes(h, B, L, C.byref(whole)) == 0
                assert whole.value == P.whole_call_workspace_bytes(cfg, B, L)
                if L == 931 and n <= 64:
                    assert got < whole.value / 8, (B, n, L)


@pytest.mark.gpu          # fs2_hifigan_create needs a device; the checks themselves run on the host
def test_window_workspace_refuses_sizes_over_the_row_limits(handles):
    lib = _lib.load()
    h3, h32 = handles["v3", _lib.MATH_3XTF32], handles["v3", _lib.MATH_FP32]
    for B, n in ((0, 4), (2, 0), (1, -3)):
        assert _ws(lib, h3, B, n)[0] == -1 and b"n_frames" in lib.fs2_last_error()
    # V3: B * (256 n + 104) < 2^31
    n = ((1 << 31) - 104 + 255) // 256
    assert _ws(lib, h3, 1, n)[0] == -1 and b"int32" in lib.fs2_last_error()
    assert _ws(lib, h3, 1, n - 1)[0] == 0
    # fp32: at most 65535 * 128 rows
    n = (65535 * 128 - 104) // 256
    assert _ws(lib, h32, 1, n)[0] == 0 and _ws(lib, h32, 1, n + 1)[0] == -1 and b"fp32" in lib.fs2_last_error()
    assert _ws(lib, h3, 1, n + 1)[0] == 0
    assert lib.fs2_hifigan_window_workspace_bytes(h3, 1, 1, None) == -1


# ---- C arguments ----------------------------------------------------------------------------------------------------
def test_window_entries_refuse_a_null_handle():
    lib = _lib.load()
    p = 256
    assert lib.fs2_hifigan_window_workspace_bytes(None, 1, 1, C.byref(C.c_size_t())) == -1 and b"null" in lib.fs2_last_error()
    assert lib.fs2_hifigan_window(None, p, p, p, 1, 8, 1, p, 256, p, p, 1 << 30, None) == -1 and b"null" in lib.fs2_last_error()


@pytest.mark.gpu          # fs2_hifigan_create needs a device; the checks themselves run on the host
def test_window_entry_rejects_bad_arguments_on_the_host(handles):
    """fs2_hifigan_window refuses these before it touches memory (the pointers are never dereferenced), in this order:
    null, alignment, window size, Lmax, audio_ld, workspace, loaded weights."""
    lib = _lib.load()
    h = handles["v3", _lib.MATH_3XTF32]
    p = 256
    big = 1 << 40

    def call(m=h, mels=p, olens=p, starts=p, B=2, L=40, n=8, audio=p, ld=8 * 256, status=p, ws=p, ws_bytes=big):
        return lib.fs2_hifigan_window(m, mels, olens, starts, B, L, n, audio, ld, status, ws, ws_bytes, None)

    for kw in ({"m": None}, {"mels": None}, {"olens": None}, {"starts": None}, {"audio": None}, {"status": None}, {"ws": None}):
        assert call(**kw) == -1 and b"null" in lib.fs2_last_error(), kw
    assert call(mels=p + 4) == -1 and b"aligned" in lib.fs2_last_error()
    for n in (0, -1):
        assert call(n=n) == -1 and b"n_frames" in lib.fs2_last_error()
    assert call(B=0) == -1 and b"n_frames" in lib.fs2_last_error()
    assert call(L=0) == -1 and b"Lmax" in lib.fs2_last_error()
    assert call(L=(1 << 31) // 256) == -1 and b"Lmax" in lib.fs2_last_error()
    assert call(ld=8 * 256 - 1) == -1 and b"audio_ld" in lib.fs2_last_error()
    need = P.workspace_bytes(P.hifigan(CONFIGS["v3"]), 2, 8)
    assert call(ws_bytes=need - 257) == -4 and b"workspace" in lib.fs2_last_error()
    # everything else valid (a row pitch above n_frames * 256 included): only the unloaded weights are left
    assert call(ws_bytes=need, ld=9 * 256) == -1 and b"not loaded" in lib.fs2_last_error()
    h32 = handles["v3", _lib.MATH_FP32]
    assert call(m=h32, B=40, n=901) == -1 and b"fp32" in lib.fs2_last_error()


def test_window_size_limits_in_python():
    v = HiFiGANVocoder("v3")
    with pytest.raises(ValueError, match="n_frames"):
        v._check_window_size(2, 0)
    with pytest.raises(ValueError, match="2\\^31"):
        v._check_window_size(1, (1 << 31) // 256)
    with pytest.raises(ValueError, match="fp32"):
        HiFiGANVocoder("v3", math_mode="fp32")._check_window_size(40, 901)
    HiFiGANVocoder("v3", math_mode="fp32")._check_window_size(40, 64)
    # a batch the whole call refuses in fp32 passes the window's limit
    f32 = HiFiGANVocoder("v1", math_mode="fp32")
    with pytest.raises(ValueError, match="fp32"):
        f32._check_size(40, 901)
    f32._check_window_size(40, 32)


# ---- Python arguments -----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def voc():
    return HiFiGANVocoder("v3")


@pytest.mark.parametrize("shape,olens,match", [
    ((2, 10), [10, 9], "mels"), ((2, 10, 40), [10, 9], "mels"), ((0, 10, 80), [], "mels"), ((2, 10, 80), [10], "olens"),
    ((2, 10, 80), [10.0, 9.0], "integer"), ((2, 10, 80), [10, 9], "CUDA")])
def test_window_bad_inputs_raise(voc, shape, olens, match):
    with pytest.raises(ValueError, match=match):
        voc.window(torch.zeros(shape), torch.tensor(olens), 0, 4)
    with pytest.raises(ValueError, match=match):
        voc(torch.zeros(shape), torch.tensor(olens), chunk_frames=4)


@pytest.mark.parametrize("starts,match", [([0], "B=2"), ([[0, 1]], "B=2"), ([0.0, 1.0], "integer"), ([-1, 0], ">= 0"),
                                          (-2, ">= 0"), ("ab", "starts"), (True, "starts")])
def test_window_bad_starts_raise(voc, starts, match):
    with pytest.raises(ValueError, match=match):
        voc._starts(torch.tensor(starts) if isinstance(starts, list) and starts and isinstance(starts[0], float) else starts, 2,
                    torch.device("cpu"))


@pytest.mark.parametrize("k", [0, -1, 2.5, None, True])
def test_chunk_frames_must_be_a_positive_int(voc, k):
    mels, olens = torch.zeros(2, 10, 80), torch.tensor([10, 9])
    if k is None:
        with pytest.raises(ValueError, match="n_frames"):
            voc.window(mels, olens, 0, k)
        return
    with pytest.raises(ValueError, match="chunk_frames"):
        voc(mels, olens, chunk_frames=k)
    with pytest.raises(ValueError, match="chunk_frames"):
        next(voc.stream(mels, olens, chunk_frames=k))
    with pytest.raises(ValueError, match="n_frames"):
        voc.window(mels, olens, 0, k)


def test_status_table_names_bad_starts(voc):
    bits = [bit for bit, _ in voc._status_table()]
    assert bits == [_lib.FS2_HIFIGAN_BAD_LENGTH, _lib.FS2_HIFIGAN_BAD_START, _lib.FS2_HIFIGAN_RANGE]


def test_library_exports_the_window_entry_points():
    lib = _lib.load()
    header = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    for name in ("fs2_hifigan_window_workspace_bytes", "fs2_hifigan_window"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES, name
        assert f"int {name}(" in header, name
    assert "#define FS2_HIFIGAN_BAD_START 4" in header and _lib.FS2_HIFIGAN_BAD_START == 4


# ---- the GPU case table ---------------------------------------------------------------------------------------------
def test_case_table_reaches_unaligned_window_starts_at_every_level():
    """The GPU window cases (tests/test_gpu_hifigan_stream.py) start windows at rows that are not multiples of 16 (where
    the level allows it) nor of 128, at every level of V1 and V3: a row then sits at another position of its GEMM tile
    than in the whole call.  And they cover starts at 0, inside the left halo, interior, near and at olens, and past it."""
    import test_gpu_hifigan_stream as G
    assert G.check_coverage() == []

