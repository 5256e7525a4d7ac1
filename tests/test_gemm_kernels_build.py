"""Build-report checks for the tensor-core tap GEMM (no GPU needed)."""
import glob
import os
import re

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _report(name):
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", name))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    return open(reports[0]).read()


def test_tap_gemm_kernels_do_not_spill():
    """Each consumer warpgroup of the ping-pong tap GEMM holds the accumulators of a whole 128 x BN tile (BN fp32 registers
    per thread) under its setmaxnreg budget; a spill would put local-memory traffic between wgmma groups."""
    text = _report("gemm_tc.ptxas.txt")
    props = re.findall(r"Function properties for (\S*tap_gemm_tc_kernel\S*)\n(.*)", text)
    # tile widths 16, 32, 64, 80, 128 in each of the tf32, f16 and 3xF16 families
    assert len(props) == 15, [name for name, _ in props]
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)


def test_no_serialized_wgmma():
    """ptxas serializes every wgmma of a kernel (warning C7510) when it cannot prove the accumulator registers untouched
    between groups, e.g. across a function call."""
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "*.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    for path in reports:
        assert "C7510" not in open(path).read(), path
