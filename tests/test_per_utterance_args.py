"""Host side of the per-utterance mode (`synthesize`, `_forward(..., per_utterance=True)`): argument validation, the
loud failure on CPU tensors, and the C entry points it runs on.  No GPU needed."""
import os

import pytest
import torch

from conftest import REPO
from fastspeech2_b200 import FeedForwardTransformer, _lib
from fastspeech2_b200.hparams import load_hp


@pytest.fixture(scope="module")
def model(weights):
    m = FeedForwardTransformer(68, 80, load_hp())
    m.load_state_dict(weights, strict=True)
    return m.eval()


def batch():
    xs = torch.zeros(3, 12, dtype=torch.int64)
    xs[:, :5] = 7
    return xs


@pytest.mark.parametrize("ilens", [[12, 0, 5], [12, -3, 5], [13, 4, 5]])
def test_ilens_out_of_range_raise(model, ilens):
    with pytest.raises(ValueError, match=r"ilens\[b\] must lie in \[1, Tmax=12\]"):
        model.synthesize(batch(), torch.tensor(ilens))
    with pytest.raises(ValueError, match="ilens"):
        model._forward(batch(), torch.tensor(ilens), is_inference=True, per_utterance=True)


def test_shape_mismatch_raises(model):
    with pytest.raises(ValueError, match="ilens must be"):
        model.synthesize(batch(), torch.tensor([12, 4]))
    with pytest.raises(ValueError, match=r"xs must be \[B, Tmax\]"):
        model.synthesize(batch()[0], torch.tensor([12]))


def test_cpu_tensors_raise(model):
    with pytest.raises(_lib.Fs2Error, match="no CPU fallback"):
        model.synthesize(batch(), torch.tensor([12, 4, 5]))


def test_library_exports_flagged_entry_points():
    lib = _lib.load()
    for name in ("fs2_encode_ex", "fs2_decode_ex", "fs2_encode", "fs2_decode"):
        assert hasattr(lib, name), name
    header = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    assert "#define FS2_PER_UTTERANCE 1" in header and _lib.FS2_PER_UTTERANCE == 1
    assert "int fs2_encode_ex(" in header and "int fs2_decode_ex(" in header
