"""The fused train attention without a GPU (DESIGN.md §13): train_attention / FS2_TRAIN_ATTENTION resolution, the new
C entries in the header, the library and _lib, their argument checks (called with fake pointers that are never
dereferenced), the workspace formula, MaskSource's (seed, offset) hand-off, and the kernels' build report."""
import ctypes as C
import glob
import os
import re

import pytest

from fastspeech2_b200 import FeedForwardTransformer, _lib
from fastspeech2_b200 import train as T
from fastspeech2_b200.hparams import load_hp

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FS2_ERR_INVALID = -1
ENTRIES = ("fs2_attn_train_ws_bytes", "fs2_attn_train_forward", "fs2_attn_train_backward")
FAKE = 1 << 20


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    monkeypatch.delenv("FS2_TRAIN_ATTENTION", raising=False)
    monkeypatch.delenv("FS2_TRAIN_PRECISION", raising=False)


# ---- interface ----------------------------------------------------------------------------------------------------------------
def test_default_is_materialized():
    assert FeedForwardTransformer(68, 80, load_hp()).train_attention == "materialized"
    assert FeedForwardTransformer(68, 80, load_hp(), train_precision="tf32").train_attention == "materialized"


def test_argument_and_environment(monkeypatch):
    assert FeedForwardTransformer(68, 80, load_hp(), train_precision="tf32", train_attention="flash").train_attention == "flash"
    monkeypatch.setenv("FS2_TRAIN_ATTENTION", "flash")
    assert FeedForwardTransformer(68, 80, load_hp(), train_precision="tf32").train_attention == "flash"
    assert FeedForwardTransformer(68, 80, load_hp(), train_precision="tf32", train_attention="materialized").train_attention == "materialized"
    monkeypatch.setenv("FS2_TRAIN_PRECISION", "tf32")
    assert FeedForwardTransformer(68, 80, load_hp()).train_attention == "flash"     # both from the environment


def test_flash_needs_tf32(monkeypatch):
    with pytest.raises(ValueError, match="1xTF32"):
        FeedForwardTransformer(68, 80, load_hp(), train_attention="flash")
    with pytest.raises(ValueError, match="1xTF32"):
        FeedForwardTransformer(68, 80, load_hp(), train_precision="fp32", train_attention="flash")
    monkeypatch.setenv("FS2_TRAIN_ATTENTION", "flash")
    with pytest.raises(ValueError, match="train_precision='tf32'"):
        FeedForwardTransformer(68, 80, load_hp())


@pytest.mark.parametrize("mode", ["Flash", "fused", "fp32", "tf32"])
def test_unknown_values_are_refused(mode, monkeypatch):
    with pytest.raises(ValueError, match="train_attention"):
        FeedForwardTransformer(68, 80, load_hp(), train_precision="tf32", train_attention=mode)
    monkeypatch.setenv("FS2_TRAIN_ATTENTION", mode)
    with pytest.raises(ValueError, match="train_attention"):
        FeedForwardTransformer(68, 80, load_hp(), train_precision="tf32")


def test_other_head_widths_are_refused():
    hp = load_hp()
    hp.model.aheads = 4                       # 256 / 4 = 64, 384 / 4 = 96
    assert FeedForwardTransformer(68, 80, hp, train_precision="tf32").train_attention == "materialized"
    with pytest.raises(ValueError, match="head widths"):
        FeedForwardTransformer(68, 80, hp, train_precision="tf32", train_attention="flash")


def test_from_checkpoint_passes_train_attention(weights):
    m = FeedForwardTransformer.from_checkpoint({"model": weights}, hp=load_hp(), train_precision="tf32", train_attention="flash")
    assert (m.train_precision, m.train_attention) == ("tf32", "flash")
    assert FeedForwardTransformer.from_checkpoint({"model": weights}, hp=load_hp()).train_attention == "materialized"
    with pytest.raises(ValueError, match="1xTF32"):
        FeedForwardTransformer.from_checkpoint({"model": weights}, hp=load_hp(), train_attention="flash")


def test_new_entry_points_are_exported():
    lib = _lib.load()
    hdr = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    for name in ENTRIES:
        assert name in _lib.SIGNATURES and hasattr(lib, name)
        assert re.search(rf"\bint {name}\(", hdr), name
    assert "4 * align256(B L C 4) + align256(B heads L 4)" in hdr


# ---- workspace formula and argument checks --------------------------------------------------------------------------------
def align256(n):
    return (n + 255) // 256 * 256


def formula(B, L, C_, heads):
    return 4 * align256(B * L * C_ * 4) + align256(B * heads * L * 4)


def lib_ws(B, L, C_, heads):
    n = C.c_size_t(0)
    rc = _lib.load().fs2_attn_train_ws_bytes(B, L, C_, heads, C.byref(n))
    return rc, int(n.value)


@pytest.mark.parametrize("case", [(1, 1, 256, 2), (5, 63, 256, 2), (3, 129, 384, 2), (64, 800, 384, 2), (64, 100, 256, 2), (8, 3200, 384, 2),
                                  (1, 8192, 384, 2), (7, 5, 128, 1), (2, 33, 576, 3)])
def test_workspace_formula(case):
    assert lib_ws(*case) == (0, formula(*case))
    assert T.attn_train_ws_bytes(*case) == formula(*case)


@pytest.mark.parametrize("args", [(0, 10, 256, 2), (1, 0, 256, 2), (-1, 10, 256, 2), (1, 10, 256, 0), (1, 10, 255, 2), (1, 10, 256, 4),
                                  (1, 10, 64, 1), (1, 10, 320, 2), (1, 10, 0, 1), (1, 10, 384, 5), (1 << 30, 1 << 30, 384, 2),
                                  (1, 1 << 30, 384, 2), (1 << 30, 4, 256, 2)])
def test_bad_or_overflowing_sizes_are_invalid(args):
    assert lib_ws(*args)[0] == FS2_ERR_INVALID
    lib = _lib.load()
    B, L, C_, heads = args
    assert lib.fs2_attn_train_forward(FAKE, FAKE, FAKE, FAKE, B, L, C_, heads, 0.0, None, 0, 0, FAKE, FAKE, FAKE, 1 << 40, None) == FS2_ERR_INVALID
    assert lib.fs2_attn_train_backward(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, B, L, C_, heads, 0.0, None, 0, 0, FAKE, FAKE, FAKE, FAKE, 1 << 40,
                                       None) == FS2_ERR_INVALID


def _fwd(**kw):
    a = dict(q=FAKE, k=FAKE, v=FAKE, lens=FAKE, B=2, L=45, C=384, heads=2, p=0.1, dmask=None, seed=0, offset=0, out=FAKE, lse=FAKE, ws=FAKE,
             ws_bytes=formula(2, 45, 384, 2))
    a.update(kw)
    return _lib.load().fs2_attn_train_forward(*a.values(), None)


def _bwd(**kw):
    a = dict(q=FAKE, k=FAKE, v=FAKE, out=FAKE, lse=FAKE, dout=FAKE, lens=FAKE, B=2, L=45, C=384, heads=2, p=0.1, dmask=None, seed=0, offset=0,
             dq=FAKE, dk=FAKE, dv=FAKE, ws=FAKE, ws_bytes=formula(2, 45, 384, 2))
    a.update(kw)
    return _lib.load().fs2_attn_train_backward(*a.values(), None)


@pytest.mark.parametrize("name", ["q", "k", "v", "lens", "out", "lse", "ws"])
def test_forward_null_pointers_are_invalid(name):
    assert _fwd(**{name: None}) == FS2_ERR_INVALID


@pytest.mark.parametrize("name", ["q", "k", "v", "out", "lse", "dout", "lens", "dq", "dk", "dv", "ws"])
def test_backward_null_pointers_are_invalid(name):
    assert _bwd(**{name: None}) == FS2_ERR_INVALID


@pytest.mark.parametrize("p", [-0.1, 1.0, 1.5, float("nan")])
def test_dropout_rate_outside_unit_interval_is_invalid(p):
    assert _fwd(p=p) == FS2_ERR_INVALID and _bwd(p=p) == FS2_ERR_INVALID


def test_short_or_misaligned_workspace_is_invalid():
    need = formula(2, 45, 384, 2)
    for call in (_fwd, _bwd):
        assert call(ws_bytes=need - 1) == FS2_ERR_INVALID
        assert b"needed" in _lib.load().fs2_last_error()
        assert call(ws=FAKE + 4) == FS2_ERR_INVALID
        assert call(ws=FAKE + 8) == FS2_ERR_INVALID


# ---- MaskSource --------------------------------------------------------------------------------------------------------------------
def test_mask_source_hands_out_the_offset_next_would_use():
    m = T.MaskSource(seed=77)
    m.offset = 5
    shape = (3, 2, 11, 11)                    # 726 elements: not a multiple of 4
    mask, seed, off = m.attention(shape, 0.2, "cpu")
    assert mask is None and (seed, off) == (77, 5)
    assert m.offset == 5 + (726 + 3) // 4 and m.calls == 1


def test_mask_source_injected_masks_pass_through():
    import torch
    inj = [torch.ones(1, 2, 3, 3, dtype=torch.bool)]
    m = T.MaskSource(injected=inj)
    mask, seed, off = m.attention((1, 2, 3, 3), 0.2, "cpu")
    assert mask.dtype == torch.uint8 and tuple(mask.shape) == (1, 2, 3, 3) and (seed, off) == (0, 0)
    assert m.offset == 0 and not m.injected


# ---- build report ----------------------------------------------------------------------------------------------------------------
def test_fused_attention_kernels_do_not_spill():
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "attention_train_tc.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = open(reports[0]).read()
    props = re.findall(r"Function properties for (\S*attn_\w+kernel\S*)\n(.*)", text)
    names = {re.search(r"attn_\w+?kernel", n).group(0) + ("<192>" if "Li192E" in n else "<128>" if "Li128E" in n else "") for n, _ in props}
    assert names == {"attn_round_kernel", "attn_delta_kernel", "attn_fwd_kernel<128>", "attn_fwd_kernel<192>", "attn_dkdv_kernel<128>",
                     "attn_dkdv_kernel<192>", "attn_dq_kernel<128>", "attn_dq_kernel<192>"}, names
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)
