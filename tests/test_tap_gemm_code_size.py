"""SASS size of every tap-GEMM instantiation in the built gemm_tc.o (cuobjdump -sass, no GPU needed).

The staged epilogue (DESIGN.md §3) keeps the kernel's code small: per tile, a warpgroup streams its epilogue once, and
the unrolled per-element epilogue it replaced was 120-180 KB of straight-line code per 3xF16 instantiation.  The
3xF16 tiles of the decoder (128 and 80 columns) must stay within 40 KB, and no instantiation may grow past its size
before the staged epilogue (f16 / tf32 at 128 columns keep the register epilogue: their ring leaves no room to stage).
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "fastspeech2_b200", "build", "gemm_tc.o")

# bytes of SASS per <BN, PRECISE, HALF> before the staged epilogue (cuobjdump -sass of the nvcc 12.9 build)
BEFORE = {
    (128, 0, 0): 143872, (128, 0, 1): 177152, (128, 1, 1): 177792,
    (80, 0, 0): 101120, (80, 0, 1): 121856, (80, 1, 1): 122624,
    (64, 0, 0): 84992, (64, 0, 1): 101760, (64, 1, 1): 102144,
    (32, 0, 0): 57984, (32, 0, 1): 63744, (32, 1, 1): 70656,
    (16, 0, 0): 40192, (16, 0, 1): 43520, (16, 1, 1): 50432,
}
STAGED_3XF16_LIMIT = 40 * 1024


def _sass_sizes(obj):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    assert os.path.exists(OBJ), f"{OBJ} missing: build the library first (python -m fastspeech2_b200.build)"
    out = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    sizes, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = None
            k = re.search(r"tap_gemm_tc_kernelILi(\d+)ELb(\d)ELb(\d)E", m.group(1))
            if k:
                cur = tuple(int(x) for x in k.groups())
                sizes[cur] = 0
            continue
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/", line)
        if m and cur is not None:
            sizes[cur] = max(sizes[cur], int(m.group(1), 16) + 16)
    return sizes


def test_every_instantiation_is_present_and_no_larger_than_before():
    sizes = _sass_sizes(OBJ)
    assert set(sizes) == set(BEFORE)
    grown = {k: (sizes[k], BEFORE[k]) for k in BEFORE if sizes[k] > BEFORE[k]}
    assert not grown, f"instantiations larger than before (bytes now, before): {grown}"


@pytest.mark.parametrize("bn", [128, 80])
def test_decoder_3xf16_tiles_are_compact(bn):
    size = _sass_sizes(OBJ)[(bn, 1, 1)]
    assert size <= STAGED_3XF16_LIMIT, f"<{bn}, 3xF16> is {size} bytes of SASS"
