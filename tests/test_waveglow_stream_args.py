"""Windowed WaveGlow without a GPU: the window plan (tests/_waveglow_window_plan.py) against the float64 oracle's NaN
dependency cone, the window workspace against fs2_waveglow_window_workspace_bytes, argument validation of the C entry
point and of `WaveGlowVocoder.window / stream / forward(chunk_frames=)`, the GPU case table's coverage and the ptxas
report of the new kernels."""
import ctypes as C
import glob
import os
import re

import pytest
import torch

import _waveglow_window_plan as P
from conftest import REPO
from fastspeech2_b200 import _lib
from fastspeech2_b200.waveglow import HALO, WaveGlowVocoder
from oracle import waveglow_oracle as O


# ---- the reach: the plan against the oracle's dependency cone -------------------------------------------------------
def test_plan_numbers_from_the_layer_shapes():
    assert [P.layer_reach(i) for i in range(8)] == [1, 2, 4, 8, 16, 32, 64, 128]
    assert P.flow_reach() == 255 and P.total_reach() == 3060 and P.cond_reach() == 3059
    assert P.halo() == HALO == 96 and P.mel_reach() == (99, 96) and P.cond_mel_reach() == (3, 0)
    assert P.plan_is_exact() and P.exact_margin(12) == 3060 <= 96 * 32
    assert P.buffer_frames(32) == 224
    # margins inside a flow: layer i's input at 255 j + 2^i - 1, its output at 255 j + 2^(i+1) - 1; the next flow starts
    # where the last layer ends
    for j in range(12):
        for i in range(8):
            assert P.exact_margin(j, i, "in") == 255 * j + 2 ** i - 1
            assert P.exact_margin(j, i, "out") == 255 * j + 2 ** (i + 1) - 1
        assert P.exact_margin(j, 7, "out") == P.exact_margin(j + 1)


def test_plan_buffers_sit_inside_the_utterance():
    assert P.buffer(0, 32, 10) == (0, 10, 0, 10)                # both sides are utterance edges
    assert P.buffer(200, 32, 1000) == (104, 328, 200, 232)      # interior: full halos
    assert P.buffer(50, 32, 1000) == (0, 178, 50, 82)           # left edge only
    assert P.buffer(990, 32, 1000) == (894, 1000, 990, 1000)    # right edge only
    assert P.buffer(1000, 4, 1000) is None and P.buffer(1200, 4, 1000) is None
    for s, n, o in ((0, 1, 1), (3, 5, 40), (97, 32, 900), (890, 32, 900), (400, 128, 931)):
        f0, f1, c0, c1 = P.buffer(s, n, o)
        assert 0 <= f0 <= c0 < c1 <= f1 <= o and f1 - f0 <= P.buffer_frames(n)
        lo, hi = P.mel_reach()
        assert f0 - 3 >= s - lo and f1 <= s + n + hi


def _oracle(C=64, seed=0):
    torch.manual_seed(seed)
    g = O.WaveGlow(C)
    with torch.no_grad():
        for name, p in g.named_parameters():
            if name.endswith("weight_g"):
                p.mul_(torch.rand(p.shape) + 0.5)
        for wn in g.WN:
            wn.end.weight.normal_(0, 1.0 / C ** 0.5)          # non-zero: a zero `end` makes every coupling the identity
            wn.end.bias.normal_(0, 0.1)
    return g.double().eval()


@pytest.fixture(scope="module")
def cone_case():
    g = _oracle()
    gen = torch.Generator().manual_seed(1)
    T = 200
    mel = torch.randn(1, 80, T, generator=gen, dtype=torch.float64) * 2 - 6
    z = torch.randn(1, 8, T * 32, generator=gen, dtype=torch.float64)
    return g, mel, z


def _nan_steps(audio):
    """[lo, hi) step rows holding a NaN sample, checked to be contiguous."""
    rows = torch.isnan(audio.reshape(-1, 8)).any(1).nonzero().flatten()
    lo, hi = int(rows.min()), int(rows.max()) + 1
    assert rows.numel() == hi - lo
    return lo, hi


def test_z_nan_cone_is_the_total_reach(cone_case):
    """NaN in every channel of one z step reaches exactly +-3060 step rows of audio (NaN * 0 = NaN: the cone is
    structural, so the equality is exact)."""
    g, mel, z = cone_case
    t0 = 3200
    zz = z.clone()
    zz[0, :, t0] = float("nan")
    with torch.no_grad():
        audio = g.infer(mel, 1.0, zz)[0]
    assert _nan_steps(audio) == (t0 - P.total_reach(), t0 + P.total_reach() + 1)


def test_mel_nan_cone_is_cond_frames_then_the_cond_reach(cone_case):
    """NaN in one mel frame f reaches cond frames f .. f + 3, then +-3059 step rows: inside the window's +-3060."""
    g, mel, z = cone_case
    f = 100
    mm = mel.clone()
    mm[0, :, f] = float("nan")
    with torch.no_grad():
        cond = g._cond(mm, mel.shape[2] * 32)
        audio = g.infer(mm, 1.0, z)[0]
    rows = torch.isnan(cond[0]).any(0).nonzero().flatten()
    left, right = P.cond_mel_reach()
    assert (int(rows.min()), int(rows.max()) + 1) == ((f - right) * 32, (f + left + 1) * 32)
    assert _nan_steps(audio) == ((f - right) * 32 - P.cond_reach(), (f + left + 1) * 32 + P.cond_reach())
    assert P.cond_reach() <= P.total_reach()


# ---- the workspace --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def handle():
    lib = _lib.load()
    hs = {}
    for mode, C_ in ((_lib.MATH_FP32, 256), (_lib.MATH_3XTF32, 512), (_lib.MATH_3XTF32, 64), (_lib.MATH_F16, 256)):
        h = C.c_void_p()
        _lib.check(lib.fs2_waveglow_create(C.byref(h), mode, C_), "fs2_waveglow_create")
        hs[(mode, C_)] = h.value
    yield hs
    for h in hs.values():
        lib.fs2_waveglow_destroy(h)


def _ws(lib, h, B, n):
    out = C.c_size_t()
    rc = lib.fs2_waveglow_window_workspace_bytes(h, B, n, C.byref(out))
    return rc, out.value


@pytest.mark.gpu          # fs2_waveglow_create needs a device; the checks themselves run on the host
def test_window_workspace_is_the_shared_plan_and_independent_of_lmax(handle):
    lib = _lib.load()
    for (mode, C_), h in handle.items():
        planes = mode != _lib.MATH_FP32
        for B, n in ((1, 1), (1, 32), (7, 13), (64, 32), (64, 64), (64, 128)):
            rc, got = _ws(lib, h, B, n)
            assert rc == 0 and got == P.workspace_bytes(C_, planes, B, n), (mode, C_, B, n)
        for B, L in ((1, 5), (64, 931)):
            whole = C.c_size_t()
            assert lib.fs2_waveglow_workspace_bytes(h, B, L, C.byref(whole)) == 0
            assert whole.value == P.whole_call_workspace_bytes(C_, planes, B, L), (mode, C_, B, L)
    # 739,584 bytes per frame at C = 512 in the plane modes: the whole filelist64 call against a 64 x 32-frame window
    assert P.whole_call_workspace_bytes(512, True, 1, 1000) - P.whole_call_workspace_bytes(512, True, 1, 999) == 739584


@pytest.mark.gpu          # fs2_waveglow_create needs a device; the checks themselves run on the host
def test_window_workspace_refuses_sizes_over_the_row_limits(handle):
    lib = _lib.load()
    h3, h32 = handle[(_lib.MATH_3XTF32, 512)], handle[(_lib.MATH_FP32, 256)]
    for B, n in ((0, 4), (2, 0), (1, -3)):
        assert _ws(lib, h3, B, n)[0] == -1 and b"n_frames" in lib.fs2_last_error()
    n = (1 << 31) // 32 - 192                                # B * (n + 192) * 32 < 2^31
    assert _ws(lib, h3, 1, n)[0] == -1 and b"int32" in lib.fs2_last_error()
    assert _ws(lib, h3, 1, n - 1)[0] == 0
    n = 65535 * 128 // 32 - 192                              # fp32: at most 65535 * 128 rows
    assert _ws(lib, h32, 1, n)[0] == 0 and _ws(lib, h32, 1, n + 1)[0] == -1 and b"fp32" in lib.fs2_last_error()
    assert _ws(lib, h3, 1, n + 1)[0] == 0


# ---- C arguments ----------------------------------------------------------------------------------------------------
def test_window_entries_refuse_a_null_handle():
    lib = _lib.load()
    p = 256
    assert lib.fs2_waveglow_window_workspace_bytes(None, 1, 1, C.byref(C.c_size_t())) == -1 and b"null" in lib.fs2_last_error()
    assert lib.fs2_waveglow_window(None, p, p, p, 1, 8, 1, 1.0, p, None, p, 256, p, p, 1 << 30, None) == -1
    assert b"null" in lib.fs2_last_error()


@pytest.mark.gpu          # fs2_waveglow_create needs a device; the checks themselves run on the host
def test_window_entry_rejects_bad_arguments_on_the_host(handle):
    """fs2_waveglow_window refuses these before it touches memory (the pointers are never dereferenced), in this order:
    null (neither seeds nor z included), alignment, sigma, window size, Lmax, audio_ld, workspace, loaded weights."""
    lib = _lib.load()
    h = handle[(_lib.MATH_3XTF32, 512)]
    p = 256
    big = 1 << 40

    def call(m=h, mels=p, olens=p, starts=p, B=2, L=40, n=8, sigma=1.0, seeds=p, z=None, audio=p, ld=8 * 256, status=p, ws=p,
             ws_bytes=big):
        return lib.fs2_waveglow_window(m, mels, olens, starts, B, L, n, sigma, seeds, z, audio, ld, status, ws, ws_bytes, None)

    for kw in ({"m": None}, {"mels": None}, {"olens": None}, {"starts": None}, {"audio": None}, {"status": None}, {"ws": None},
               {"seeds": None}):
        assert call(**kw) == -1 and b"null" in lib.fs2_last_error(), kw
    assert call(mels=p + 4) == -1 and b"aligned" in lib.fs2_last_error()
    for sigma in (float("nan"), float("inf"), -0.5):
        assert call(sigma=sigma) == -1 and b"sigma" in lib.fs2_last_error(), sigma
    for n in (0, -1):
        assert call(n=n) == -1 and b"n_frames" in lib.fs2_last_error()
    assert call(B=0) == -1 and b"n_frames" in lib.fs2_last_error()
    assert call(n=(1 << 31) // 64) == -1 and b"int32" in lib.fs2_last_error()
    assert call(L=0) == -1 and b"Lmax" in lib.fs2_last_error()
    assert call(L=(1 << 31) // 32) == -1 and b"Lmax" in lib.fs2_last_error()
    assert call(ld=8 * 256 - 1) == -1 and b"audio_ld" in lib.fs2_last_error()
    need = P.workspace_bytes(512, True, 2, 8)
    assert call(ws_bytes=need - 257) == -4 and b"workspace" in lib.fs2_last_error()
    # everything else valid (z in place of seeds, a row pitch above n_frames * 256): only the unloaded weights are left
    assert call(ws_bytes=need, ld=9 * 256, seeds=None, z=p) == -1 and b"not loaded" in lib.fs2_last_error()
    # fp32: the window's rows, not Lmax, meet the limit -- a batch the whole call refuses takes small windows
    h32 = handle[(_lib.MATH_FP32, 256)]
    assert call(m=h32, B=40, n=6400) == -1 and b"fp32" in lib.fs2_last_error()
    ws = C.c_size_t()
    assert lib.fs2_waveglow_workspace_bytes(h32, 40, 6600, C.byref(ws)) == -1
    assert lib.fs2_waveglow_window_workspace_bytes(h32, 40, 64, C.byref(ws)) == 0


def test_window_size_limits_in_python():
    v = WaveGlowVocoder(256)
    with pytest.raises(ValueError, match="n_frames"):
        v._check_window_size(2, 0)
    with pytest.raises(ValueError, match="2\\^31"):
        v._check_window_size(1, (1 << 31) // 32 - 192)
    v._check_window_size(1, (1 << 31) // 32 - 193)
    f = WaveGlowVocoder(256, math_mode="fp32")
    with pytest.raises(ValueError, match="fp32"):
        f._check_window_size(1, 65535 * 128 // 32 - 191)
    f._check_window_size(1, 65535 * 128 // 32 - 192)
    f._check_window_size(40, 64)
    with pytest.raises(ValueError, match="fp32"):
        f._check_size(40, 6600)                               # the whole call refuses what the windows take


# ---- Python arguments -----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def voc():
    return WaveGlowVocoder(64)


@pytest.mark.parametrize("shape,olens,match", [
    ((2, 10), [10, 9], "mels"), ((2, 10, 40), [10, 9], "mels"), ((0, 10, 80), [], "mels"), ((2, 10, 80), [10], "olens"),
    ((2, 10, 80), [10.0, 9.0], "integer"), ((2, 10, 80), [10, 9], "CUDA")])
def test_window_bad_inputs_raise(voc, shape, olens, match):
    with pytest.raises(ValueError, match=match):
        voc.window(torch.zeros(shape), torch.tensor(olens), 0, 4, seed=1)
    with pytest.raises(ValueError, match=match):
        voc(torch.zeros(shape), torch.tensor(olens), chunk_frames=4, seed=1)
    with pytest.raises(ValueError, match=match):
        next(voc.stream(torch.zeros(shape), torch.tensor(olens), 4, seed=1))


@pytest.mark.parametrize("kw,match", [
    (dict(sigma=float("nan"), seed=1), "sigma"), (dict(sigma=-1.0, seed=1), "sigma"),
    (dict(z=torch.zeros(2, 8, 319)), "z must be"), (dict(z=torch.zeros(2, 8, 320), seed=1), "either z or seed"),
    (dict(seed=torch.tensor([1, 2, 3])), "seed"), (dict(seed=1.5), "seed"), (dict(seed=True), "seed")])
def test_window_bad_noise_arguments_raise(voc, kw, match):
    with pytest.raises(ValueError, match=match):
        voc.window(torch.zeros(2, 10, 80), torch.tensor([10, 9]), 0, 4, **kw)


def test_window_refuses_seed_none(voc):
    """A window is only meaningful against a whole call with the same noise, so it never draws its own."""
    with pytest.raises(ValueError, match="noise"):
        voc.window(torch.zeros(2, 10, 80), torch.tensor([10, 9]), 0, 4)
    with pytest.raises(ValueError, match="noise"):
        voc.window(torch.zeros(2, 10, 80), torch.tensor([10, 9]), 0, 4, seed=None, z=None)


def test_stream_and_chunked_forward_draw_the_whole_calls_seed():
    """seed=None: one int64 from torch's CPU generator, as forward draws it, drawn once for every window."""
    torch.manual_seed(9)
    want = int(torch.randint(-2 ** 63, 2 ** 63 - 1, (), dtype=torch.int64))
    torch.manual_seed(9)
    assert WaveGlowVocoder._resolve_seed(None, None) == want
    torch.manual_seed(9)
    assert torch.equal(WaveGlowVocoder._seeds(None, 3, "cpu"), torch.arange(3) + want)
    assert WaveGlowVocoder._resolve_seed(None, torch.zeros(1)) is None and WaveGlowVocoder._resolve_seed(5, None) == 5


@pytest.mark.parametrize("starts,match", [([0], "B=2"), ([[0, 1]], "B=2"), ([0.0, 1.0], "integer"), ([-1, 0], ">= 0"),
                                          (-2, ">= 0"), ("ab", "starts"), (True, "starts")])
def test_window_bad_starts_raise(voc, starts, match):
    with pytest.raises(ValueError, match=match):
        voc._starts(torch.tensor(starts) if isinstance(starts, list) and starts and isinstance(starts[0], float) else starts, 2,
                    torch.device("cpu"))


def test_window_host_starts_become_an_int64_vector(voc):
    for s in (3, [3, 3], torch.tensor([3, 3], dtype=torch.int32)):
        out = voc._starts(s, 2, torch.device("cpu"))
        assert out.dtype == torch.int64 and out.tolist() == [3, 3]


@pytest.mark.parametrize("k", [0, -1, 2.5, None, True])
def test_chunk_frames_must_be_a_positive_int(voc, k):
    mels, olens = torch.zeros(2, 10, 80), torch.tensor([10, 9])
    if k is None:
        with pytest.raises(ValueError, match="n_frames"):
            voc.window(mels, olens, 0, k, seed=1)
        return
    with pytest.raises(ValueError, match="chunk_frames"):
        voc(mels, olens, chunk_frames=k)
    with pytest.raises(ValueError, match="chunk_frames"):
        next(voc.stream(mels, olens, chunk_frames=k))
    with pytest.raises(ValueError, match="n_frames"):
        voc.window(mels, olens, 0, k, seed=1)


def test_library_exports_the_window_entry_points():
    lib = _lib.load()
    header = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    for name in ("fs2_waveglow_window_workspace_bytes", "fs2_waveglow_window"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES, name
        assert f"int {name}(" in header, name
    assert "#define FS2_WAVEGLOW_BAD_START 4" in header and _lib.FS2_WAVEGLOW_BAD_START == 4
    assert "It enqueues 497 kernels (498 in FS2_MATH_F16 / FS2_MATH_3XTF32)" in header


# ---- the GPU case table ---------------------------------------------------------------------------------------------
def test_case_table_reaches_every_window_shape():
    """The GPU window cases (tests/test_gpu_waveglow_stream.py) reach windows at both utterance edges, at one edge only,
    interior with full halos on both sides, starts at or past olens, and buffer first rows at every 32-row residue mod
    128 (so that rows sit at other tile positions than in the whole call) with ragged buffer tails."""
    import test_gpu_waveglow_stream as G
    assert G.check_coverage() == []


# ---- ptxas ----------------------------------------------------------------------------------------------------------
def test_window_audio_kernel_does_not_spill():
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "waveglow.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = open(reports[0]).read()
    props = re.findall(r"Function properties for \S*wg_win_audio_kernel\S*\n(.*)", text)
    assert len(props) == 1, len(props)
    assert "0 bytes spill stores, 0 bytes spill loads" in props[0], props[0]
    props = re.findall(r"Function properties for (\S*wg_\S*)\n(.*)", text)
    assert len(props) == 18 + 1                            # the whole call's 18 instantiations and the window's audio copy
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)
