"""Windowed MelGAN without a GPU: the window plan (tests/_melgan_window_plan.py) against the float64 oracle's dependency
cone, the window workspace against fs2_melgan_window_workspace_bytes, argument validation of the C entry point and of
`MelGANVocoder.window / stream / forward(chunk_frames=)`, the GPU case table's coverage and the ptxas report."""
import ctypes as C
import glob
import os
import re

import pytest
import torch

import _melgan_window_plan as P
from conftest import REPO
from fastspeech2_b200 import _lib
from fastspeech2_b200.melgan import MelGANVocoder
from oracle import melgan_oracle as O


# ---- the reach: the plan against the oracle's dependency cone -------------------------------------------------------
def _generator():
    torch.manual_seed(0)
    return O.Generator().double().eval()


def _levels(gen, mel):
    """Forward of the oracle's layers, keeping each layer's input: [('conv0', mel frames), ('convt0', ...), ('res0', ...),
    ..., ('post', the last conv's input), ('audio', ...)], each [1, C, rows]."""
    seq = gen.generator
    x = (mel + 5.0) / 5.0
    out = [("conv0", x)]
    x = seq[1](seq[0](x))
    for s, i in enumerate((3, 6, 9, 12)):
        out.append((f"convt{s}", x))
        x = seq[i](seq[i - 1](x))
        out.append((f"res{s}", x))
        x = seq[i + 1](x)
    out.append(("post", x))
    out.append(("audio", seq[17](seq[16](seq[15](seq[14](x))))))
    return out


def _rate(name):
    if name in ("conv0", "convt0"):
        return 1
    if name == "post":
        return 256
    s = int(name[-1])
    return P.UP[s] if name.startswith("convt") else P.UP[s + 1]


# (frames of the whole input incl. the 10 tail frames, chunk [c0, c1)): interior chunks of 1, 4 and 13 frames, a chunk at
# the left edge, one ending at olens (c1 = frames - 10), and a 1-frame utterance
CONE_CASES = [(30, 14, 15), (30, 12, 16), (40, 13, 26), (24, 0, 3), (24, 9, 14), (11, 0, 1)]


@pytest.mark.parametrize("frames,c0,c1", CONE_CASES)
def test_plan_reach_is_the_oracle_backprop_cone(frames, c0, c1):
    """Back-propagating a random functional of the chunk's audio gives, at every layer's input, nonzero gradients on
    exactly the plan's window (clipped to the utterance): every row of the plan changes some sample, no other row does."""
    gen = _generator()
    g = torch.Generator().manual_seed(frames + c0)
    mel = (torch.randn(1, 80, frames, generator=g, dtype=torch.float64) * 2 - 6).requires_grad_(True)
    levels = _levels(gen, mel)
    for _, t in levels[1:-1]:
        t.retain_grad()
    audio = levels[-1][1]
    w = torch.randn(audio[0, 0, c0 * 256: c1 * 256].shape, generator=g, dtype=torch.float64)
    (audio[0, 0, c0 * 256: c1 * 256] * w).sum().backward()
    reach = P.reaches()
    for name, t in levels[:-1]:
        grad = mel.grad if name == "conv0" else t.grad
        rows = (grad[0].abs().sum(0) != 0).nonzero().flatten()
        up, n = _rate(name), frames * _rate(name)
        want = (max(c0 * up - reach[name], 0), min(c1 * up + reach[name], n))
        assert (int(rows.min()), int(rows.max()) + 1) == want, (name, frames, c0, c1)
        assert rows.numel() == want[1] - want[0], name                        # contiguous


def test_plan_reach_matches_the_nan_cone():
    """A NaN mel frame just outside [c0 - 6, c1 + 6) leaves the chunk's audio finite; one just inside reaches it."""
    gen = _generator()
    c0, c1, frames = 15, 19, 34
    r = P.reaches()["conv0"]
    assert r == 6
    base = torch.randn(1, 80, frames, generator=torch.Generator().manual_seed(3), dtype=torch.float64) * 2 - 6
    for f, inside in ((c0 - r - 1, False), (c0 - r, True), (c1 + r - 1, True), (c1 + r, False)):
        mel = base.clone()
        mel[0, :, f] = float("nan")
        with torch.no_grad():
            audio = gen(mel)[0, 0, c0 * 256: c1 * 256]
        assert bool(torch.isnan(audio).any()) == inside, f
    # one NaN frame's cone: +-1425 samples around its own 256
    mel = base.clone()
    mel[0, :, 16] = float("nan")
    with torch.no_grad():
        nan = torch.isnan(gen(mel)[0, 0]).nonzero().flatten()
    assert (int(nan.min()), int(nan.max()) + 1) == (16 * 256 - 1425, 17 * 256 + 1425)


def test_plan_layout_is_exact_and_as_documented():
    assert P.reaches() == {"conv0": 6, "convt0": 3, "res0": 17, "convt1": 4, "res1": 25, "convt2": 12, "res2": 22,
                           "convt3": 9, "res3": 16, "post": 3}
    assert [P.level_halo(s) for s in range(5)] == [3, 24, 32, 24, 18]
    for s, margin, room in P.exact_margins():
        assert margin <= room, s
    for s in range(4):
        assert P.level_rows(s + 1, 7) == P.STRIDES[s] * P.convt_rows(s, 7)
    assert P.level_rows(4, 32) == 256 * 32 + 36
    # every buffer of a window lies inside its level's rows, and the next layer's window inside it
    for start, n, olens in ((0, 1, 1), (3, 5, 40), (17, 32, 900), (890, 32, 900)):
        w = P.windows(start, n, olens)
        lvl = {s: w[f"level{s}"] for s in range(5)}
        for s in range(5):
            assert lvl[s][1] - lvl[s][0] <= P.level_rows(s, n)
            assert lvl[s][1] < (olens + 10) * P.UP[s]                      # the right side is never the utterance's edge
        for s in range(1, 4):
            lo, hi = w[f"convt{s}"]
            assert lvl[s][0] <= lo and hi <= lvl[s][1] and hi - lo <= P.convt_rows(s, n)


# ---- the workspace --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def handle():
    lib = _lib.load()
    hs = {}
    for mode in (_lib.MATH_FP32, _lib.MATH_3XTF32):
        h = C.c_void_p()
        _lib.check(lib.fs2_melgan_create(C.byref(h), mode), "fs2_melgan_create")
        hs[mode] = h.value
    yield hs
    for h in hs.values():
        lib.fs2_melgan_destroy(h)


def _ws(lib, h, B, n):
    out = C.c_size_t()
    rc = lib.fs2_melgan_window_workspace_bytes(h, B, n, C.byref(out))
    return rc, out.value


@pytest.mark.gpu          # fs2_melgan_create needs a device; the checks themselves run on the host
def test_window_workspace_is_the_plan_and_smaller_than_the_whole_call(handle):
    lib = _lib.load()
    h = handle[_lib.MATH_3XTF32]
    for B, n in ((1, 1), (1, 32), (7, 13), (64, 16), (64, 32), (64, 64), (3, 901)):
        rc, got = _ws(lib, h, B, n)
        assert rc == 0 and got == P.workspace_bytes(B, n), (B, n)
        for L in (n + 1, 2 * n, 931):
            if n < L:
                whole = C.c_size_t()
                assert lib.fs2_melgan_workspace_bytes(h, B, L, C.byref(whole)) == 0
                assert whole.value == P.whole_call_workspace_bytes(B, L)
                assert got < whole.value, (B, n, L)
    assert abs(P.workspace_bytes(64, 32) / 1e9 - 0.415) < 0.001


@pytest.mark.gpu          # fs2_melgan_create needs a device; the checks themselves run on the host
def test_window_workspace_refuses_sizes_over_the_row_limits(handle):
    lib = _lib.load()
    h3, h32 = handle[_lib.MATH_3XTF32], handle[_lib.MATH_FP32]
    for B, n in ((0, 4), (2, 0), (1, -3)):
        assert _ws(lib, h3, B, n)[0] == -1 and b"n_frames" in lib.fs2_last_error()
    # B * (256 n + 36) < 2^31
    n = ((1 << 31) - 36 + 255) // 256
    assert _ws(lib, h3, 1, n)[0] == -1 and b"int32" in lib.fs2_last_error()
    assert _ws(lib, h3, 1, n - 1)[0] == 0
    # fp32: at most 65535 * 128 rows
    n = (65535 * 128 - 36) // 256
    assert _ws(lib, h32, 1, n)[0] == 0 and _ws(lib, h32, 1, n + 1)[0] == -1 and b"fp32" in lib.fs2_last_error()
    assert _ws(lib, h3, 1, n + 1)[0] == 0
    assert lib.fs2_melgan_window_workspace_bytes(None, 1, 1, C.byref(C.c_size_t())) == -1
    assert lib.fs2_melgan_window_workspace_bytes(h3, 1, 1, None) == -1


# ---- C arguments ----------------------------------------------------------------------------------------------------
def test_window_entries_refuse_a_null_handle():
    lib = _lib.load()
    p = 256
    assert lib.fs2_melgan_window_workspace_bytes(None, 1, 1, C.byref(C.c_size_t())) == -1 and b"null" in lib.fs2_last_error()
    assert lib.fs2_melgan_window(None, p, p, p, 1, 8, 1, p, 256, p, p, 1 << 30, None) == -1 and b"null" in lib.fs2_last_error()


@pytest.mark.gpu          # fs2_melgan_create needs a device; the checks themselves run on the host
def test_window_entry_rejects_bad_arguments_on_the_host(handle):
    """fs2_melgan_window refuses these before it touches memory (the pointers are never dereferenced), in this order:
    null, alignment, window size, Lmax, audio_ld, workspace, loaded weights."""
    lib = _lib.load()
    h = handle[_lib.MATH_3XTF32]
    p = 256
    big = 1 << 40

    def call(m=h, mels=p, olens=p, starts=p, B=2, L=40, n=8, audio=p, ld=8 * 256, status=p, ws=p, ws_bytes=big):
        return lib.fs2_melgan_window(m, mels, olens, starts, B, L, n, audio, ld, status, ws, ws_bytes, None)

    for kw in ({"m": None}, {"mels": None}, {"olens": None}, {"starts": None}, {"audio": None}, {"status": None}, {"ws": None}):
        assert call(**kw) == -1 and b"null" in lib.fs2_last_error(), kw
    assert call(mels=p + 4) == -1 and b"aligned" in lib.fs2_last_error()
    for n in (0, -1):
        assert call(n=n) == -1 and b"n_frames" in lib.fs2_last_error()
    assert call(B=0) == -1 and b"n_frames" in lib.fs2_last_error()
    assert call(L=0) == -1 and b"Lmax" in lib.fs2_last_error()
    assert call(L=(1 << 31) // 256) == -1 and b"Lmax" in lib.fs2_last_error()
    assert call(ld=8 * 256 - 1) == -1 and b"audio_ld" in lib.fs2_last_error()
    need = P.workspace_bytes(2, 8)
    assert call(ws_bytes=need - 257) == -4 and b"workspace" in lib.fs2_last_error()
    # everything else valid (a row pitch above n_frames * 256 included): only the unloaded weights are left
    assert call(ws_bytes=need, ld=9 * 256) == -1 and b"not loaded" in lib.fs2_last_error()
    h32 = handle[_lib.MATH_FP32]
    assert call(m=h32, B=40, n=901) == -1 and b"fp32" in lib.fs2_last_error()


def test_window_size_limits_in_python():
    v = MelGANVocoder()
    with pytest.raises(ValueError, match="n_frames"):
        v._check_window_size(2, 0)
    with pytest.raises(ValueError, match="2\\^31"):
        v._check_window_size(1, (1 << 31) // 256)
    with pytest.raises(ValueError, match="fp32"):
        MelGANVocoder(math_mode="fp32")._check_window_size(40, 901)
    MelGANVocoder(math_mode="fp32")._check_window_size(40, 64)


# ---- Python arguments -----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def voc():
    return MelGANVocoder()


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


def test_window_host_starts_become_an_int64_vector(voc):
    for s in (3, [3, 3], torch.tensor([3, 3], dtype=torch.int32)):
        out = voc._starts(s, 2, torch.device("cpu"))
        assert out.dtype == torch.int64 and out.tolist() == [3, 3]


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


def test_library_exports_the_window_entry_points():
    lib = _lib.load()
    header = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    for name in ("fs2_melgan_window_workspace_bytes", "fs2_melgan_window"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES, name
        assert f"int {name}(" in header, name
    assert "#define FS2_MELGAN_BAD_START 4" in header and _lib.FS2_MELGAN_BAD_START == 4


# ---- the GPU case table ---------------------------------------------------------------------------------------------
def test_case_table_reaches_unaligned_window_starts_at_every_level():
    """The GPU window cases (tests/test_gpu_melgan_stream.py) start windows at rows that are not multiples of 16 (where
    the level allows it) nor of 128, at every level: a row then sits at another position of its GEMM tile than in the
    whole call.  And they cover starts at 0, inside the left halo, interior, near and at olens, and past it."""
    import test_gpu_melgan_stream as G
    assert G.check_coverage() == []


# ---- ptxas ----------------------------------------------------------------------------------------------------------
def test_window_support_adds_no_instantiation_and_no_spill():
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "melgan.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = open(reports[0]).read()
    props = re.findall(r"Function properties for (\S*melgan\S*)\n(.*)", text)
    assert len(props) == 1 + 1 + 1 + 1 + 3 + 3 + 6 + 8                    # as before windows: runtime arguments only
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)
