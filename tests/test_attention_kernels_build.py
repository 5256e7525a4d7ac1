"""Build-report checks for the attention kernels (no GPU needed)."""
import glob
import os
import re

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_wgmma_attention_kernels_do_not_spill():
    """The warp-specialised attention keeps O (d_k / 2 fp32), S, P hi / lo and the softmax statistics in registers; a
    spill would put local-memory traffic between every pair of wgmma groups."""
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "attention_tc.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = open(reports[0]).read()
    props = re.findall(r"Function properties for (\S*attention_wgmma_kernel\S*)\n(.*)", text)
    # d_k 128 (encoder) and 192 (decoder), each f16 and 3xF16
    assert len(props) == 4, [name for name, _ in props]
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)
