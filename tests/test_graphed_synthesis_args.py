"""Graphed synthesis without a device: the capacity plan's C entry is declared, bound and exported, the C entries refuse
bad arguments before touching the device, and `graphed_synthesize` / `GraphedSynthesis` refuse what they cannot capture
or serve."""
import os
import re
import subprocess

import pytest
import torch

from conftest import REPO
from fastspeech2_b200 import FeedForwardTransformer, _lib
from fastspeech2_b200.fastspeech import GraphedSynthesis
from fastspeech2_b200.hparams import load_hp
from fastspeech2_b200.vocoder import GriffinLimVocoder

FAKE = 0x1000      # a non-null pointer the entries must refuse before they dereference it


@pytest.mark.parametrize("name", ["fs2_length_plan_cap", "fs2_synth_status"])
def test_declared_bound_and_exported(name):
    with open(os.path.join(REPO, "include", "fs2_b200.h")) as f:
        assert re.search(rf"\bint {name}\(", f.read())
    assert name in _lib.SIGNATURES
    nm = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert re.search(rf"\bT {name}$", nm, re.M)
    assert callable(getattr(_lib.load(), name))


def test_status_bits_match_the_header():
    with open(os.path.join(REPO, "include", "fs2_b200.h")) as f:
        h = f.read()
    for name in ("FS2_PLAN_BAD_ILENS", "FS2_PLAN_BAD_CONTROL", "FS2_PLAN_OVERFLOW", "FS2_SYNTH_VOC_SHIFT"):
        assert int(re.search(rf"#define {name} (\d+)", h).group(1)) == getattr(_lib, name), name


def _plan_cap(**kw):
    a = dict(ds=FAKE, dtype=_lib.FS2_DUR_I64, ilens=FAKE, alpha_v=None, fac=None, B=2, T=5, Lc=100, cum=FAKE, olens=FAKE,
             need=FAKE, d_used=None, status=FAKE)
    a.update(kw)
    rc = _lib.load().fs2_length_plan_cap(a["ds"], a["dtype"], a["ilens"], a["alpha_v"], a["fac"], a["B"], a["T"], a["Lc"], a["cum"],
                                         a["olens"], a["need"], a["d_used"], a["status"], None)
    return rc, _lib.load().fs2_last_error().decode()


@pytest.mark.parametrize("kw, match", [
    ({"ds": None}, "null argument"),
    ({"ilens": None}, "null argument"),
    ({"cum": None}, "null argument"),
    ({"olens": None}, "null argument"),
    ({"need": None}, "null argument"),
    ({"status": None}, "null argument"),
    ({"B": 0}, r"B=0 and Tmax=5 must be >= 1"),
    ({"T": 0}, r"B=2 and Tmax=0 must be >= 1"),
    ({"Lc": 0}, r"capacity Lc=0 must lie in \[1, 2147483647\]"),
    ({"Lc": -5}, r"capacity Lc=-5"),
    ({"Lc": 2 ** 31}, r"capacity Lc=2147483648 must lie in \[1, 2147483647\] \(the prefix sum is int32\)"),
])
def test_plan_cap_host_refusals(kw, match):
    rc, msg = _plan_cap(**kw)
    assert rc == -1
    assert re.search(match, msg), msg


def test_synth_status_host_refusals():
    lib = _lib.load()
    assert lib.fs2_synth_status(None, None, FAKE, 2, 256, FAKE, None, None) == -1
    assert "null argument" in lib.fs2_last_error().decode()
    assert lib.fs2_synth_status(FAKE, None, FAKE, 0, 256, FAKE, None, None) == -1
    assert "B=0" in lib.fs2_last_error().decode()


@pytest.fixture(scope="module")
def model():
    return FeedForwardTransformer(68, 80, load_hp()).eval()


@pytest.mark.parametrize("args, match", [
    ((2, 10, 0), "capacity must be an int >= 1"),
    ((2, 10, -3), "capacity must be an int >= 1"),
    ((2, 10, 1.5), "capacity must be an int >= 1"),
    ((0, 10, 100), "B must be an int >= 1"),
    ((2, 0, 100), "T must be an int >= 1"),
    ((2, 10, 2 ** 31), "exceeds the length plan's int32 prefix sum"),
])
def test_capture_refuses_bad_sizes(model, args, match):
    with pytest.raises(ValueError, match=match):
        model.graphed_synthesize(*args)


@pytest.mark.parametrize("vocoder", [object(), GriffinLimVocoder()])
def test_capture_refuses_what_is_not_a_neural_vocoder(model, vocoder):
    with pytest.raises(ValueError, match="vocoder must be a NeuralVocoder upsampling chain"):
        model.graphed_synthesize(2, 10, 100, vocoder=vocoder)


def test_capture_refuses_waveglow(model):
    from fastspeech2_b200.waveglow import WaveGlowVocoder
    with pytest.raises(ValueError, match="WaveGlow's noise and Griffin-Lim are not captured"):
        model.graphed_synthesize(2, 10, 100, vocoder=WaveGlowVocoder.__new__(WaveGlowVocoder))


def test_capture_needs_the_model_on_the_gpu(model):
    with pytest.raises(_lib.Fs2Error, match="no CPU fallback"):
        model.graphed_synthesize(2, 10, 100)


@pytest.mark.parametrize("xs, ilens, match", [
    (torch.ones(5, 4, dtype=torch.long), torch.full((5,), 4), r"b=5 utterances of t=4 phonemes does not fit the graph's B=4, T=8"),
    (torch.ones(2, 9, dtype=torch.long), torch.full((2,), 9), r"b=2 utterances of t=9 phonemes does not fit the graph's B=4, T=8"),
    (torch.ones(2, 4, dtype=torch.long), torch.full((3,), 4), r"ilens must be a \[b=2\] tensor"),
    (torch.ones(2, 4, dtype=torch.long), torch.full((2,), 4.0), "ilens must be an integer tensor"),
    (torch.ones(2, 4, dtype=torch.long), torch.tensor([4, 5]), r"every ilens\[b\] must lie in \[0, t=4\]"),
    (torch.ones(2, 4, dtype=torch.long), torch.tensor([-1, 2]), r"every ilens\[b\] must lie in \[0, t=4\]"),
    (torch.ones(4, dtype=torch.long), torch.full((1,), 4), r"xs must be a non-empty \[b, t\] tensor"),
    (torch.ones(0, 4, dtype=torch.long), torch.full((0,), 4), r"xs must be a non-empty \[b, t\] tensor"),
])
def test_request_refusals(xs, ilens, match):
    with pytest.raises(ValueError, match=match):
        GraphedSynthesis.check_request(xs, ilens, 4, 8)


def test_request_that_fits():
    assert GraphedSynthesis.check_request(torch.ones(3, 6, dtype=torch.long), torch.tensor([6, 0, 2]), 4, 8) == (3, 6)
