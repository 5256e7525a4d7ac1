"""The deterministic train mode without a GPU (DESIGN.md §26): how the flag resolves, the aligner's CLI flag, the argument
checks of every `_det` entry (refused with FS2_ERR_INVALID before anything is launched), each `_ws_bytes` answer against
tests/_det_plan.py, and a SASS scan of the built library: the ordered instantiations hold no floating-point atomic, and
the kernels that do are exactly the default path's."""
import inspect
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch

import _det_plan as D
import _train_plan as P
from fastspeech2_b200 import FeedForwardTransformer, _lib
from fastspeech2_b200 import aligner as A
from fastspeech2_b200 import train as T
from fastspeech2_b200.fastspeech import resolve_train_deterministic
from fastspeech2_b200.hparams import load_hp
from fastspeech2_b200._kernel_module import query_bytes

FS2_ERR_INVALID = -1
FAKE = 1 << 20           # a non-null, 16-byte aligned pointer that is never dereferenced
WS_BIG = 1 << 40


# ---- the flag ------------------------------------------------------------------------------------------------------------------
def test_flag_resolution(monkeypatch):
    monkeypatch.delenv("FS2_TRAIN_DETERMINISTIC", raising=False)
    assert resolve_train_deterministic() is False
    assert resolve_train_deterministic(True) is True
    for v, want in (("1", True), ("true", True), ("ON", True), ("0", False), ("", False), ("off", False)):
        monkeypatch.setenv("FS2_TRAIN_DETERMINISTIC", v)
        assert resolve_train_deterministic() is want, v
    monkeypatch.setenv("FS2_TRAIN_DETERMINISTIC", "1")
    assert resolve_train_deterministic(False) is False           # the argument wins over the environment
    monkeypatch.setenv("FS2_TRAIN_DETERMINISTIC", "maybe")
    with pytest.raises(ValueError, match="FS2_TRAIN_DETERMINISTIC"):
        resolve_train_deterministic()
    with pytest.raises(ValueError, match="train_deterministic"):
        resolve_train_deterministic(1)


def test_model_flag_and_torch_flag(monkeypatch):
    monkeypatch.delenv("FS2_TRAIN_DETERMINISTIC", raising=False)
    off = FeedForwardTransformer(68, 80, load_hp())
    on = FeedForwardTransformer(68, 80, load_hp(), train_deterministic=True)
    assert off.train_deterministic is False and on.train_deterministic is True
    monkeypatch.setenv("FS2_TRAIN_DETERMINISTIC", "1")
    assert FeedForwardTransformer(68, 80, load_hp()).train_deterministic is True
    explicit_off = FeedForwardTransformer(68, 80, load_hp(), train_deterministic=False)
    assert explicit_off.train_deterministic is False
    assert T.deterministic_step(on) and not T.deterministic_step(explicit_off)
    was = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        assert T.deterministic_step(explicit_off)            # train_deterministic=False does not override torch's flag
    finally:
        torch.use_deterministic_algorithms(was)
    assert not T.deterministic_step(explicit_off)


def test_from_checkpoint_passes_the_flag(monkeypatch):
    monkeypatch.delenv("FS2_TRAIN_DETERMINISTIC", raising=False)
    from fastspeech2_b200 import synthetic_state_dict
    m = FeedForwardTransformer.from_checkpoint(synthetic_state_dict(0), hp=load_hp(), train_deterministic=True)
    assert m.train_deterministic is True
    assert "train_deterministic" in inspect.signature(FeedForwardTransformer.from_checkpoint).parameters


def test_aligner_cli_flag(monkeypatch, tmp_path):
    seen = {}
    assert inspect.signature(A.train).parameters["deterministic"].default is False

    def fake_train(corpus, n_symbols, steps, batch=32, bin_start=None, **kw):
        seen.update(kw)
        return A.Aligner(n_symbols), []

    monkeypatch.setattr(A, "train", fake_train)
    monkeypatch.setattr(A, "Corpus", lambda lines, symbols, data_dir, log=None: object())
    monkeypatch.setattr(A, "read_filelist", lambda path: [])
    monkeypatch.setattr(A, "build_symbols", lambda lines: ["_", "a"])
    monkeypatch.setattr(A, "save", lambda *a, **k: None)
    cfg = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "fastspeech2_b200", "configs", "default.yaml")
    if not os.path.exists(cfg):
        pytest.skip("no default config in the tree")
    base = ["train", "-c", cfg, "--filelist", "x", "-d", str(tmp_path), "-o", str(tmp_path / "a.pt"), "--steps", "1"]
    A.main(base)
    assert seen["deterministic"] is False
    A.main(base + ["--deterministic"])
    assert seen["deterministic"] is True


# ---- argument checks ------------------------------------------------------------------------------------------------------------
def refused(fn, *args, msg=b""):
    lib = _lib.load()
    n0 = lib.fs2_kernel_launches()
    rc = getattr(lib, fn)(*args)
    assert rc == FS2_ERR_INVALID, (fn, args, rc)
    err = lib.fs2_last_error()
    assert fn.encode() in err and msg in err, err
    assert lib.fs2_kernel_launches() == n0


def test_colsum_det_refusals():
    refused("fs2_colsum_det", None, 10, 8, FAKE, FAKE, WS_BIG, None, msg=b"null")
    refused("fs2_colsum_det", FAKE, 10, 0, FAKE, FAKE, WS_BIG, None)
    refused("fs2_colsum_det", FAKE, -1, 8, FAKE, FAKE, WS_BIG, None)
    refused("fs2_colsum_det", FAKE, 10, 8, FAKE, None, WS_BIG, None, msg=b"workspace")
    refused("fs2_colsum_det", FAKE, 10, 8, FAKE, FAKE + 4, WS_BIG, None, msg=b"aligned")
    refused("fs2_colsum_det", FAKE, 10, 8, FAKE, FAKE, D.colsum_bytes(10, 8) - 1, None, msg=b"needed")


def test_conv_wgrad_det_refusals():
    good = (FAKE, FAKE, 2, 50, 80, 80, 3, FAKE, FAKE)
    for bad in ((2, 50, 80, 80, 2), (2, 50, 0, 80, 1), (-1, 50, 80, 80, 1), (2, 50, 80, 80, -1)):
        refused("fs2_conv_wgrad_det", FAKE, FAKE, *bad, FAKE, FAKE, FAKE, WS_BIG, None, msg=b"odd taps")
    refused("fs2_conv_wgrad_det", None, *good[1:], FAKE, WS_BIG, None, msg=b"null")
    refused("fs2_conv_wgrad_det", *good, FAKE, D.conv_wgrad_bytes(2, 50, 80, 80, 3) - 1, None, msg=b"needed")
    refused("fs2_conv_wgrad_det", *good, None, WS_BIG, None, msg=b"workspace")


def test_layernorm_det_refusals():
    refused("fs2_layernorm_backward_det", FAKE, FAKE, FAKE, 1e-5, 10, 320, FAKE, FAKE, FAKE, FAKE, WS_BIG, None, msg=b"C in")
    refused("fs2_layernorm_backward_det", FAKE, None, FAKE, 1e-5, 10, 256, FAKE, FAKE, FAKE, FAKE, WS_BIG, None, msg=b"null")
    refused("fs2_layernorm_backward_det", FAKE + 4, FAKE, FAKE, 1e-5, 10, 256, FAKE, FAKE, FAKE, FAKE, WS_BIG, None, msg=b"aligned")
    refused("fs2_layernorm_backward_det", FAKE, FAKE, FAKE, 1e-5, 10, 256, FAKE, FAKE, FAKE, FAKE, D.layernorm_bytes(10, 256) - 1, None,
            msg=b"needed")


def test_batchnorm_det_refusals():
    refused("fs2_batchnorm_train_det", FAKE, 0, 80, FAKE, FAKE, 1e-5, 0.1, 0, FAKE, FAKE, FAKE, FAKE, FAKE, WS_BIG, None)
    refused("fs2_batchnorm_train_det", FAKE, 10, 80, None, FAKE, 1e-5, 0.1, 0, FAKE, FAKE, FAKE, FAKE, FAKE, WS_BIG, None, msg=b"null")
    refused("fs2_batchnorm_train_det", FAKE, 10, 80, FAKE, FAKE, 1e-5, 0.1, 0, FAKE, None, FAKE, FAKE, FAKE, WS_BIG, None, msg=b"together")
    refused("fs2_batchnorm_train_det", FAKE, 10, 80, FAKE, FAKE, 1e-5, 0.1, 0, FAKE, FAKE, FAKE, FAKE, FAKE, D.batchnorm_bytes(10, 80) - 1, None,
            msg=b"needed")
    refused("fs2_batchnorm_backward_det", FAKE, FAKE, FAKE, FAKE, 1e-5, 10, 0, FAKE, FAKE, FAKE, FAKE, WS_BIG, None)
    refused("fs2_batchnorm_backward_det", FAKE, FAKE, FAKE, FAKE, 1e-5, 10, 80, FAKE, FAKE, FAKE, FAKE + 8, WS_BIG, None, msg=b"aligned")
    refused("fs2_batchnorm_backward_det", FAKE, FAKE, FAKE, FAKE, 1e-5, 10, 80, FAKE, FAKE, FAKE, FAKE, D.batchnorm_bytes(10, 80) - 1, None,
            msg=b"needed")


def test_embed_det_refusals():
    refused("fs2_embed_backward_det", None, FAKE, FAKE, 2, 5, 256, 68, FAKE, FAKE, FAKE, WS_BIG, None, msg=b"null")
    refused("fs2_embed_backward_det", FAKE, FAKE, FAKE, 2, 5, 256, 0, FAKE, FAKE, FAKE, WS_BIG, None, msg=b"n_sym")
    refused("fs2_embed_backward_det", FAKE, FAKE, FAKE, 2, 5, 256, D.SC_MAX_IDS + 1, FAKE, FAKE, FAKE, WS_BIG, None, msg=b"n_sym")
    refused("fs2_embed_backward_det", FAKE, FAKE, FAKE, -2, 5, 256, 68, FAKE, FAKE, FAKE, WS_BIG, None)
    refused("fs2_embed_backward_det", FAKE, FAKE, FAKE, 2, 5, 256, 68, FAKE, FAKE, FAKE, D.embed_bytes(2, 5, 256, 68) - 1, None, msg=b"needed")


def test_onehot_and_rowdot_det_refusals():
    refused("fs2_onehot_linear_backward_det", FAKE, None, 10, 256, 256, FAKE, FAKE, FAKE, WS_BIG, None, msg=b"null")
    refused("fs2_onehot_linear_backward_det", FAKE, FAKE, 10, 256, 0, FAKE, FAKE, FAKE, WS_BIG, None, msg=b"n_bins")
    refused("fs2_onehot_linear_backward_det", FAKE, FAKE, 1 << 31, 256, 256, FAKE, FAKE, FAKE, WS_BIG, None, msg=b"rows")
    refused("fs2_onehot_linear_backward_det", FAKE, FAKE, 10, 256, 256, FAKE, FAKE, FAKE, D.onehot_bytes(10, 256, 256) - 1, None, msg=b"needed")
    refused("fs2_rowdot_backward_det", FAKE, FAKE, FAKE, None, 10, 5, 400, FAKE, FAKE, FAKE, FAKE, WS_BIG, None, msg=b"C <= 384")
    refused("fs2_rowdot_backward_det", FAKE, FAKE, FAKE, None, 10, 0, 256, FAKE, FAKE, FAKE, FAKE, WS_BIG, None, msg=b"L > 0")
    refused("fs2_rowdot_backward_det", FAKE, FAKE, FAKE, None, 10, 5, 256, FAKE, None, FAKE, FAKE, WS_BIG, None, msg=b"null")
    refused("fs2_rowdot_backward_det", FAKE, FAKE, FAKE, None, 10, 5, 256, FAKE, FAKE, FAKE, FAKE, D.rowdot_bytes(10, 256) - 1, None,
            msg=b"needed")


def test_masked_losses_det_refusals():
    args = [FAKE] * 3 + [100, FAKE, FAKE, 0] + [FAKE] * 6 + [2, 10, 100, 80, FAKE]
    refused("fs2_masked_losses_det", *args, FAKE, D.loss_bytes(2, 10, 100, 80) - 1, None, msg=b"needed")
    bad = list(args); bad[16] = 82
    refused("fs2_masked_losses_det", *bad, FAKE, WS_BIG, None, msg=b"multiple of 4")
    bad = list(args); bad[2] = FAKE + 4
    refused("fs2_masked_losses_det", *bad, FAKE, WS_BIG, None, msg=b"aligned")
    bad = list(args); bad[11] = None
    refused("fs2_masked_losses_det", *bad, FAKE, WS_BIG, None, msg=b"null")


def test_size_queries_refuse_bad_shapes():
    lib = _lib.load()
    import ctypes
    n = ctypes.c_size_t(0)
    assert lib.fs2_colsum_det_ws_bytes(10, 0, ctypes.byref(n)) == FS2_ERR_INVALID
    assert lib.fs2_conv_wgrad_det_ws_bytes(1, 10, 80, 80, 2, ctypes.byref(n)) == FS2_ERR_INVALID
    assert lib.fs2_layernorm_backward_det_ws_bytes(10, 320, ctypes.byref(n)) == FS2_ERR_INVALID
    assert lib.fs2_embed_backward_det_ws_bytes(2, 5, 256, D.SC_MAX_IDS + 1, ctypes.byref(n)) == FS2_ERR_INVALID
    assert lib.fs2_colsum_det_ws_bytes(10, 8, None) == FS2_ERR_INVALID


# ---- workspace sizes ------------------------------------------------------------------------------------------------------------
CONV_CASES = P.conv_cases([(256, 256, 1), (1024, 256, 9), (80, 384, 1), (256, 80, 5)]) + P.WGRAD_TAIL_CASES + [(0, 70, 80, 80, 1)]


def test_ws_bytes_match_the_plan():
    for rows in P.COLSUM_ROWS + [0]:
        for C in P.COLSUM_CS:
            assert query_bytes("fs2_colsum_det_ws_bytes", rows, C) == D.colsum_bytes(rows, C), (rows, C)
    for case in CONV_CASES:
        assert query_bytes("fs2_conv_wgrad_det_ws_bytes", *case) == D.conv_wgrad_bytes(*case), case
    for rows in P.LN_ROWS + [0]:
        for C in P.LN_CS:
            assert query_bytes("fs2_layernorm_backward_det_ws_bytes", rows, C) == D.layernorm_bytes(rows, C), (rows, C)
            assert query_bytes("fs2_rowdot_backward_det_ws_bytes", rows, C) == D.rowdot_bytes(rows, C), (rows, C)
    for rows in P.BN_ROWS:
        for C in P.BN_CS:
            assert query_bytes("fs2_batchnorm_train_det_ws_bytes", rows, C) == D.batchnorm_bytes(rows, C)
            assert query_bytes("fs2_batchnorm_backward_det_ws_bytes", rows, C) == D.batchnorm_bytes(rows, C)
    for B, T_, C, n in ((64, 100, 384, 68), (64, 800, 384, 0), (1, 1, 256, 2), (0, 5, 256, 68), (3, 70, 256, D.SC_MAX_IDS)):
        assert query_bytes("fs2_embed_backward_det_ws_bytes", B, T_, C, n) == D.embed_bytes(B, T_, C, n)
    for rows, C, nb in ((51200, 384, 256), (1, 256, 256), (0, 384, 256), (4225, 384, 1)):
        assert query_bytes("fs2_onehot_linear_backward_det_ws_bytes", rows, C, nb) == D.onehot_bytes(rows, C, nb)
    for B, T_, L, odim in ((64, 100, 800, 80), (2, 24, 190, 80), (0, 1, 1, 80), (3, 400, 17, 80)):
        assert query_bytes("fs2_masked_losses_det_ws_bytes", B, T_, L, odim) == D.loss_bytes(B, T_, L, odim)


def test_plan_takes_no_sm_count():
    for name, fn in inspect.getmembers(D, inspect.isfunction):
        params = [p.lower() for p in inspect.signature(fn).parameters]
        assert not any("sm" in p for p in params), name
    src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "fastspeech2_b200", "csrc", "train_det.cu")).read()
    assert "multiProcessorCount" not in src and "sm_count" not in src
    tr = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "fastspeech2_b200", "csrc", "train.cu")).read()
    assert "multiProcessorCount" not in tr and "sm_count" not in tr


def test_c2_workspace_is_small():
    """the largest ordered workspace of a c2 step (B = 64, T = 100, L = 800): the decoder-side one-hot scatter"""
    rows = P.C2_B * P.C2_L
    assert D.onehot_bytes(rows, 384, 256) < 2 << 20 and D.embed_bytes(P.C2_B, P.C2_L, 384, 0) < 2 << 20
    assert D.layernorm_bytes(rows, 384) < 4 << 20


# ---- SASS scan ------------------------------------------------------------------------------------------------------------------
FLOAT_ATOMIC = re.compile(r"\b(?:REDG|ATOMG|RED|ATOM)\.[A-Z0-9_.]*\.F(?:32|64)\b|ATOMS\.CAST\.SPIN")
RETURNING_INT_ATOMG = re.compile(r"\bATOMG\.E\.[A-Z0-9_.]*")
def sass_functions():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    filt = shutil.which("c++filt")
    if not os.path.exists(exe) or not filt:
        pytest.skip("cuobjdump / c++filt not available")
    out = subprocess.run([exe, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    parts = re.split(r"\n[ \t]+Function : (\S+)[ \t]*\n", out)
    mangled = parts[1::2]
    names = subprocess.run([filt], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout.split("\n")
    return {D.short_name(n): body for n, body in zip(names, parts[2::2])}


@pytest.fixture(scope="module")
def sass():
    return sass_functions()


def test_ordered_kernels_have_no_float_atomics(sass):
    missing = D.ORDERED - set(sass)
    assert not missing, missing
    for name in sorted(D.ORDERED):
        body = sass[name]
        assert not FLOAT_ATOMIC.search(body), (name, FLOAT_ATOMIC.search(body).group(0))
        assert not RETURNING_INT_ATOMG.search(body), (name, RETURNING_INT_ATOMG.search(body).group(0))


def test_float_atomic_kernels_are_exactly_the_default_path(sass):
    have = {name for name, body in sass.items() if FLOAT_ATOMIC.search(body)}
    assert have == D.DEFAULT_ATOMIC, (sorted(have - D.DEFAULT_ATOMIC), sorted(D.DEFAULT_ATOMIC - have))


def test_the_scan_sees_the_atomics_it_looks_for(sass):
    """the forms sm_90a emits for a global float / double atomicAdd and a shared float atomicAdd"""
    assert re.search(r"REDG\.E\.ADD\.F32\.FTZ\.RN\.STRONG\.GPU", sass["colsum_kernel<false>"])
    assert re.search(r"REDG\.E\.ADD\.F64\.RN", sass["bn_stats_kernel<false>"])
    assert "ATOMS.CAST.SPIN" in sass["layernorm_backward_kernel<2, false>"]
