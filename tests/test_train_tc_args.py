"""The tf32 train mode without a GPU: train_precision / FS2_TRAIN_PRECISION validation, the tensor-core weight-gradient
kernel's workspace formula and argument checks, what the GPU cases of tests/test_gpu_train_tc.py reach in its work
decomposition (tests/_wgrad_plan.py), and its build report."""
import ctypes as C
import glob
import os
import re

import pytest

from _wgrad_plan import H100_SMS, KERNEL_CASES, TRAIN_SHAPES, box_starts, plan, split_inside_utterance, ws_bytes
from fastspeech2_b200 import FeedForwardTransformer, _lib
from fastspeech2_b200 import train as T
from fastspeech2_b200.hparams import load_hp

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FS2_ERR_INVALID = -1


# ---- interface ------------------------------------------------------------------------------------------------------------
def test_default_is_fp32(monkeypatch):
    monkeypatch.delenv("FS2_TRAIN_PRECISION", raising=False)
    m = FeedForwardTransformer(68, 80, load_hp())
    assert m.train_precision == "fp32"
    assert FeedForwardTransformer(68, 80, load_hp(), precision="fp32").train_precision == "fp32"


def test_argument_and_environment(monkeypatch):
    monkeypatch.delenv("FS2_TRAIN_PRECISION", raising=False)
    assert FeedForwardTransformer(68, 80, load_hp(), train_precision="tf32").train_precision == "tf32"
    monkeypatch.setenv("FS2_TRAIN_PRECISION", "tf32")
    m = FeedForwardTransformer(68, 80, load_hp())
    assert m.train_precision == "tf32"
    assert FeedForwardTransformer(68, 80, load_hp(), train_precision="fp32").train_precision == "fp32"   # the argument wins
    monkeypatch.setenv("FS2_TRAIN_PRECISION", "bf16")
    with pytest.raises(ValueError, match="train_precision"):
        FeedForwardTransformer(68, 80, load_hp())


def test_precision_and_train_precision_are_independent(monkeypatch):
    monkeypatch.delenv("FS2_TRAIN_PRECISION", raising=False)
    m = FeedForwardTransformer(68, 80, load_hp(), precision="f16", train_precision="tf32")
    assert (m.precision, m.train_precision) == ("f16", "tf32")
    m = FeedForwardTransformer(68, 80, load_hp(), precision="tf32")
    assert (m.precision, m.train_precision) == ("tf32", "fp32")


@pytest.mark.parametrize("mode", ["f16", "3xf16", "3xtf32"])
def test_plane_modes_are_refused_with_the_reason(mode):
    with pytest.raises(ValueError, match="underflow"):
        FeedForwardTransformer(68, 80, load_hp(), train_precision=mode)


@pytest.mark.parametrize("mode", ["bf16", "TF32", "fp16"])
def test_unknown_modes_are_refused(mode):
    with pytest.raises(ValueError, match="train_precision"):
        FeedForwardTransformer(68, 80, load_hp(), train_precision=mode)


def test_from_checkpoint_passes_train_precision(weights, monkeypatch):
    monkeypatch.delenv("FS2_TRAIN_PRECISION", raising=False)
    m = FeedForwardTransformer.from_checkpoint({"model": weights}, hp=load_hp(), train_precision="tf32")
    assert m.train_precision == "tf32"
    assert FeedForwardTransformer.from_checkpoint({"model": weights}, hp=load_hp()).train_precision == "fp32"
    with pytest.raises(ValueError, match="underflow"):
        FeedForwardTransformer.from_checkpoint({"model": weights}, hp=load_hp(), train_precision="f16")


def test_convfn_math_mode_defaults_to_fp32():
    import inspect
    sig = inspect.signature(T.ConvFn.forward)
    assert list(sig.parameters)[-1] == "math" and sig.parameters["math"].default == _lib.MATH_FP32


def test_new_entry_points_are_exported():
    lib = _lib.load()
    for name in ("fs2_conv_forward_ex", "fs2_conv_dgrad_ex", "fs2_conv_wgrad_tc", "fs2_conv_wgrad_tc_ws_bytes"):
        assert name in _lib.SIGNATURES and hasattr(lib, name)
    hdr = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    for name in ("fs2_conv_forward_ex", "fs2_conv_dgrad_ex", "fs2_conv_wgrad_tc", "fs2_conv_wgrad_tc_ws_bytes"):
        assert re.search(rf"\bint {name}\(", hdr), name


# ---- the weight-gradient kernel's workspace and argument checks -------------------------------------------------------------
def _lib_ws(B, L, N, K, taps):
    n = C.c_size_t(0)
    rc = _lib.load().fs2_conv_wgrad_tc_ws_bytes(B, L, N, K, taps, C.byref(n))
    return rc, int(n.value)


@pytest.mark.parametrize("case", KERNEL_CASES + [(16, 800, N, K, t) for (N, K, t) in TRAIN_SHAPES] +
                         [(64, 800, N, K, t) for (N, K, t) in TRAIN_SHAPES] + [(0, 10, 80, 80, 1), (3, 0, 80, 80, 1)])
def test_workspace_formula(case):
    assert _lib_ws(*case) == (0, ws_bytes(*case))


@pytest.mark.parametrize("args", [(1, 10, 80, 80, 2), (1, 10, 80, 80, 0), (1, 10, 0, 80, 1), (1, 10, 80, 0, 1), (-1, 10, 80, 80, 1),
                                  (1, -1, 80, 80, 1), (1 << 30, 1 << 30, 1 << 20, 1 << 20, 9), (1 << 30, 4, 1 << 30, 1, 1),
                                  (1, (1 << 30) - 2, 80, 80, 9), (1, 1 << 20, 1 << 30, 80, 1)])
def test_bad_or_overflowing_sizes_are_invalid(args):
    assert _lib_ws(*args)[0] == FS2_ERR_INVALID


def test_short_or_misaligned_workspace_is_invalid():
    """Checked before anything reaches the device (the pointers below are never dereferenced)."""
    lib = _lib.load()
    B, L, N, K, taps = 2, 45, 256, 80, 5
    need = ws_bytes(B, L, N, K, taps)
    fake = 1 << 20
    assert lib.fs2_conv_wgrad_tc(fake, fake, B, L, N, K, taps, fake, None, fake, need - 1, None) == FS2_ERR_INVALID
    assert b"needed" in lib.fs2_last_error()
    assert lib.fs2_conv_wgrad_tc(fake, fake, B, L, N, K, taps, fake, None, None, need, None) == FS2_ERR_INVALID
    assert lib.fs2_conv_wgrad_tc(fake, fake, B, L, N, K, taps, fake, None, fake + 4, need, None) == FS2_ERR_INVALID
    assert lib.fs2_conv_wgrad_tc(None, fake, B, L, N, K, taps, fake, None, fake, need, None) == FS2_ERR_INVALID


def test_other_math_modes_are_invalid_in_the_ex_entries():
    lib = _lib.load()
    fake = 1 << 20
    for mode in (_lib.MATH_3XTF32, _lib.MATH_F16, 7):
        assert lib.fs2_conv_forward_ex(fake, 1, 8, 80, fake, None, 80, 1, 0, None, fake, fake, mode, None) == FS2_ERR_INVALID
        assert lib.fs2_conv_dgrad_ex(fake, 1, 8, 80, fake, 80, 1, fake, fake, mode, None) == FS2_ERR_INVALID


# ---- what the GPU cases reach -----------------------------------------------------------------------------------------------
def test_kernel_cases_cover_every_train_shape():
    assert {(N, K, t) for (_, _, N, K, t) in KERNEL_CASES} >= set(TRAIN_SHAPES)
    assert {80, 256, 384, 1024} <= {N for (N, _, _) in TRAIN_SHAPES} and {1, 3, 5, 9} == {t for (_, _, t) in TRAIN_SHAPES}


def test_kernel_cases_reach_the_decomposition_edges():
    plans = [plan(*c) for c in KERNEL_CASES]
    assert any(p["units"] <= H100_SMS for p in plans), "a case with one unit per CTA"
    assert any(p["units"] > 2 * H100_SMS for p in plans), "a case where CTAs walk more than two units"
    assert any(split_inside_utterance(*c) for c in KERNEL_CASES), "a split boundary inside an utterance"
    assert any(p["splits"] > 1 for p in plans) and any(p["splits"] == 1 for p in plans)
    Ls = [(L, t) for (_, L, _, _, t) in KERNEL_CASES]
    assert any(L == 1 for L, _ in Ls)
    assert any(L < (t - 1) // 2 for L, t in Ls), "L < pad"
    assert any(L % 4 != 0 for L, _ in Ls) and any(L % 32 != 0 and L % 4 != 0 for L, _ in Ls)
    assert any(N % 128 != 0 for (_, _, N, _, _) in KERNEL_CASES) and any(K % 128 != 0 for (_, _, _, K, _) in KERNEL_CASES)


@pytest.mark.parametrize("taps", [1, 3, 5, 9, 17])
@pytest.mark.parametrize("L", [1, 3, 45, 70, 800])
def test_x_box_starts_are_aligned_and_read_the_right_times(L, taps):
    """Copy r holds time t at column t + P + r; a box at column c reads times c - P - r ...: the time the tap wants."""
    p = plan(1, L, 128, 128, taps)
    pad = (taps - 1) // 2
    starts = box_starts(L, taps)
    assert all(c % 4 == 0 and c >= 0 and r < p["phases"] and ext <= p["Lx"] for c, r, ext in starts)
    for j in range(taps):
        for i, t0 in enumerate(range(0, L, 32)):
            c, r, _ = starts[j * len(range(0, L, 32)) + i]
            assert c - p["P"] - r == t0 + j - pad


def test_plan_splits_are_ordered_and_nonempty():
    for c in KERNEL_CASES + [(64, 800, N, K, t) for (N, K, t) in TRAIN_SHAPES]:
        p = plan(*c)
        b = p["bounds"]
        assert b[0] == 0 and b[-1] == p["Q"] and all(b1 > b0 for b0, b1 in zip(b, b[1:])), c


# ---- build report -------------------------------------------------------------------------------------------------------------
def test_wgrad_kernels_do_not_spill():
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "wgrad_tc.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = open(reports[0]).read()
    props = re.findall(r"Function properties for (\S*(?:wgrad_tc_kernel|wgrad_reduce_kernel|transpose_tf32_kernel)\S*)\n(.*)", text)
    assert len(props) == 3, [name for name, _ in props]
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)
    assert "C7510" not in text
