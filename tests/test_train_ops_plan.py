"""The fp32 train kernels without a GPU: the launch geometry restated in tests/_train_plan.py against the constants of
csrc/train.cu, what the GPU cases of tests/test_gpu_train_ops.py reach in it, that every C entry of train.cu has a GPU
test, and the argument checks that refuse a shape before anything is launched."""
import ast
import os
import re

import pytest

import _train_plan as P
from _wgrad_plan import TRAIN_SHAPES
from fastspeech2_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAIN_CU = os.path.join(REPO, "fastspeech2_b200", "csrc", "train.cu")
GPU_TESTS = os.path.join(REPO, "tests", "test_gpu_train_ops.py")
FS2_ERR_INVALID = -1


def _src():
    return open(TRAIN_CU).read()


# ---- the restatement follows train.cu ----------------------------------------------------------------------------------------
def test_plan_constants_are_train_cu_s():
    s = _src()
    assert "rows / 8 + 1 > 132 * 4 ? 132 * 4 : rows / 8 + 1" in s                 # layernorm / rowdot backward grids
    assert "rows / 512 + 1 > 64 ? 64 : rows / 512 + 1" in s                       # colsum
    assert s.count("rows / 256 + 1 > 128 ? 128 : rows / 256 + 1") == 2            # bn_stats, bn_backward_sums
    assert "int chunks = (132 * 4 + tiles - 1) / tiles;" in s and "(M + 255) / 256" in s
    assert "constexpr int WG_T = 64, WG_KM = 16;" in s and P.WG_T == 64
    assert "for (int u = lane; u < L; u += 32)" in s                              # softmax: lane strides over keys
    assert "__shared__ float sa[16][65], sb[16][65];" in s                        # bgemm: 64 x 64 tiles, K steps of 16


def test_warp_rows_regimes():
    assert P.warp_rows(4223) == (528, 0, 1)
    assert P.warp_rows(4224) == (528, 1, 1)
    assert P.warp_rows(4225) == (528, 1, 2)
    assert P.warp_rows(51200) == (528, 12, 13)
    assert P.warp_rows(1) == (1, 0, 1)


def test_wgrad_plan_at_c2():
    assert P.wgrad(64, 800, 80, 384, 1)["chunks"] == 44
    assert P.wgrad(64, 800, 384, 384, 1)["chunks"] == 15
    p = P.wgrad(64, 100, 256, 256, 1)
    assert p["chunks"] == 25 == -(-6400 // 256) and p["boundary_inside_utterance"]


# ---- what the GPU cases reach -------------------------------------------------------------------------------------------------
def test_layernorm_and_rowdot_cases_reach_every_regime():
    rpw = [P.warp_rows(r) for r in P.LN_ROWS]
    assert any(lo == hi == 1 for _, lo, hi in rpw), "one row per warp"
    assert any(hi >= 3 for _, _, hi in rpw), "several rows per warp"
    assert {4223, 4224, 4225} <= set(P.LN_ROWS)
    assert any(c < 528 for c, _, _ in rpw) and any(c == 528 for c, _, _ in rpw)
    assert max(P.warp_rows(r)[2] for r in P.ROWDOT_ROWS) > 1 and min(P.warp_rows(r)[2] for r in P.ROWDOT_ROWS) > 1
    assert 6400 in P.LN_ROWS and 51200 in P.LN_ROWS                              # the c2 encoder and decoder row counts


def test_wgrad_cases_reach_every_regime():
    cases = P.conv_cases(TRAIN_SHAPES) + P.WGRAD_TAIL_CASES
    plans = [(c, P.wgrad(*c)) for c in cases]
    chunks = {p["chunks"] for _, p in plans}
    assert 1 in chunks and 2 in chunks and max(chunks) >= 33
    capped = [(c, p) for c, p in plans if p["chunks"] == -(-(c[0] * c[1]) // 256) < -(-528 // p["tiles"])]
    assert any(p["boundary_inside_utterance"] for _, p in capped), "the ceil(M / 256) cap with a boundary inside an utterance"
    assert any(p["boundary_inside_utterance"] for _, p in plans if p["chunks"] >= 33)
    assert {(N, K, t) for (_, _, N, K, t) in cases} >= set(TRAIN_SHAPES)
    for (N, K, t) in TRAIN_SHAPES:
        assert any(c[2:] == (N, K, t) and c[:2] == (3, 70) for c in cases)
        assert any(c[2:] == (N, K, t) and c[0] == 64 and c[1] in (100, 800) for c in cases)
    assert {1, 65} <= {N for (_, _, N, _, _) in cases} and {1, 65} <= {K for (_, _, _, K, _) in cases}
    for t in (5, 9):
        pad = (t - 1) // 2
        assert {1, pad, pad + 1} <= {L for (_, L, _, _, tt) in cases if tt == t}


def test_colsum_and_bn_cases_reach_every_regime():
    gys = {P.colsum(r, 1)["grid_y"] for r in P.COLSUM_ROWS}
    assert 1 in gys and 64 in gys
    assert min(P.colsum(r, 1)["rows_per_lane"] for r in P.COLSUM_ROWS) == 1 and max(P.colsum(r, 1)["rows_per_lane"] for r in P.COLSUM_ROWS) > 1
    assert {C % 32 for C in P.COLSUM_CS} >= {0, 1, 31}
    bys = [P.bn(r)["grid_y"] for r in P.BN_ROWS]
    assert any(g < 128 for g in bys) and any(g == 128 for g in bys)
    assert any(C % 32 for C in P.BN_CS)


def test_softmax_cases_reach_every_regime():
    Ls = P.SOFTMAX_LS
    assert any(L < 32 for L in Ls) and 32 in Ls and 33 in Ls and max(Ls) >= 800
    assert any(P.softmax(L)["idle_lanes"] > 0 for L in Ls) and any(P.softmax(L)["idle_lanes"] == 0 for L in Ls)
    for L in Ls:
        lens = P.SOFTMAX_LENS(L)
        assert 0 in lens and 1 in lens and L in lens and any(n > L for n in lens)


def test_bgemm_cases_reach_every_tail():
    cases = P.bgemm_cases()
    for slot in (1, 2, 3):
        assert {1, 15, 17, 63, 65} <= {c[slot] for c in cases}, slot
    assert set(P.BGEMM_PATTERNS) == {c[0] for c in cases} and {1, 2, 3} == {c[4] for c in cases}
    tails = [P.bgemm(*c[1:4]) for c in cases]
    assert {1, 15, 17, 63} <= {t["tail_m"] for t in tails} and {1, 15, 17, 63} <= {t["tail_n"] for t in tails}
    assert {0, 1, 15} <= {t["tail_k"] for t in tails}


# ---- every train.cu entry has a GPU test -------------------------------------------------------------------------------------
def train_cu_entries():
    s = _src()
    block = s[s.index('extern "C" {'):]
    return sorted(set(re.findall(r"^int (fs2_\w+)\(", block, re.M)))


def entries_called_by_tests(src):
    """C entries the test functions of `src` call: `call("fs2_x", ...)` with a string constant, or an attribute `.fs2_x`
    (`lib().fs2_x(...)`), in a test or in any module-level helper a test reaches through calls.  Names in docstrings,
    comments or other strings do not count."""
    funcs = {f.name: f for f in ast.parse(src).body if isinstance(f, ast.FunctionDef)}
    direct, calls = {}, {}
    for name, f in funcs.items():
        d, c = set(), set()
        for n in ast.walk(f):
            if isinstance(n, ast.Call) and isinstance(n.func, ast.Name):
                c.add(n.func.id)
                if n.func.id == "call" and n.args and isinstance(n.args[0], ast.Constant) and isinstance(n.args[0].value, str):
                    d.add(n.args[0].value)
            elif isinstance(n, ast.Attribute) and n.attr.startswith("fs2_"):
                d.add(n.attr)
        direct[name], calls[name] = d, c & set(funcs)
    out = set()
    for name in funcs:
        if not name.startswith("test_"):
            continue
        seen, todo = set(), [name]
        while todo:
            f = todo.pop()
            if f not in seen:
                seen.add(f)
                out |= direct[f]
                todo += calls[f]
    return out


def test_the_coverage_matcher_counts_calls_only():
    src = ('def helper():\n    lib().fs2_b(1)\n\ndef via():\n    helper()\n\n'
           'def test_one():\n    """calls fs2_a"""\n    call("fs2_c", 1)  # fs2_d\n    x = "fs2_e"\n    via()\n\n'
           'def unreached():\n    call("fs2_f")\n')
    assert entries_called_by_tests(src) == {"fs2_b", "fs2_c"}


def test_every_train_cu_entry_has_a_gpu_test():
    names = train_cu_entries()
    assert len(names) >= 26 and "fs2_conv_wgrad" in names and "fs2_loss_backward" in names
    called = entries_called_by_tests(open(GPU_TESTS).read())
    missing = [n for n in names if n not in called]
    assert not missing, f"train.cu entries no test in tests/test_gpu_train_ops.py calls: {missing}"
    assert "fs2_masked_losses" in called


# ---- argument checks: refused before anything reaches the device --------------------------------------------------------------
FAKE = 1 << 20       # a non-null pointer that is never dereferenced


@pytest.mark.parametrize("args", [(1, 10, 80, 80, 2), (1, 10, 80, 80, 0), (1, 10, 80, 80, -3), (1, 10, 0, 80, 1), (1, 10, 80, 0, 1),
                                  (-1, 10, 80, 80, 1), (1, -1, 80, 80, 1)])
def test_conv_wgrad_refuses_bad_shapes(args):
    lib = _lib.load()
    n0 = lib.fs2_kernel_launches()
    assert lib.fs2_conv_wgrad(FAKE, FAKE, *args, FAKE, FAKE, None) == FS2_ERR_INVALID
    assert b"odd taps" in lib.fs2_last_error()
    assert lib.fs2_kernel_launches() == n0


@pytest.mark.parametrize("taps", [0, 2, 4, -1])
def test_conv_dgrad_refuses_even_taps_before_packing(taps):
    lib = _lib.load()
    n0 = lib.fs2_kernel_launches()
    assert lib.fs2_conv_dgrad(FAKE, 1, 8, 80, FAKE, 80, taps, FAKE, FAKE, None) == FS2_ERR_INVALID
    assert b"fs2_conv_dgrad: taps must be odd" in lib.fs2_last_error()
    for mode in (_lib.MATH_FP32, _lib.MATH_TF32):
        assert lib.fs2_conv_dgrad_ex(FAKE, 1, 8, 80, FAKE, 80, taps, FAKE, FAKE, mode, None) == FS2_ERR_INVALID
        assert b"taps must be odd" in lib.fs2_last_error()
    assert lib.fs2_kernel_launches() == n0
