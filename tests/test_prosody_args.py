"""Prosody controls (speed, pitch, energy) without a GPU: the CPU oracle against the reference's own modules wired with
scalar alphas (tests/golden/inf_controls.npz), the duration rule on ties and on the all-zero rule, argument validation,
and the C entry points."""
import glob
import os
import re

import numpy as np
import pytest
import torch

import _prosody_oracle as P
from conftest import REPO
from fastspeech2_b200 import FeedForwardTransformer, _lib
from fastspeech2_b200.hparams import load_hp
from test_oracle_golden import close

T_ = torch.from_numpy


def test_oracle_reproduces_reference_controls(golden, weights):
    """Same standard as inf_single: float outputs within 1e-6, integers exact."""
    g = golden("inf_controls")
    x = T_(g["x"])
    n = x.shape[0]
    torch.set_num_threads(1)
    for i, (s, p, e) in enumerate(g["cases"].tolist()):
        with torch.no_grad():
            _, after, used, e_ids, p_ids, e_val, p_val = P.inference_path(
                weights, x[None], torch.tensor([n]), P.per_phoneme(s, n), P.per_phoneme(p, n), P.per_phoneme(e, n))
        want_used = torch.round(T_(g[f"d_pred{i}"]).float() * torch.tensor(s, dtype=torch.float32)).long()
        assert torch.equal(used[0], want_used) and int(used.sum()) == g[f"mel{i}"].shape[0], i
        assert torch.equal(e_ids[0], T_(g[f"e_ids{i}"])) and torch.equal(p_ids[0], T_(g[f"p_ids{i}"])), i
        assert torch.equal(e_val[0], T_(g[f"e_val{i}"])) and torch.equal(p_val[0], T_(g[f"p_val{i}"])), i
        close(after[0], g[f"mel{i}"])


def test_cases_cover_ties_and_unrepresentable_factors(golden):
    g = golden("inf_controls")
    speeds = g["cases"][:, 0]
    assert float(np.float32(1.1)) != 1.1 and 1.1 in speeds
    d = T_(g["d_pred1"]).double() * 2.5                    # speed 2.5 on odd durations: exact halves, round to even
    assert speeds[1] == 2.5 and bool(((d % 1) == 0.5).any())


def test_duration_rule_matches_reference_length_regulator(golden):
    """Per-phoneme factors, all equal, against the reference LengthRegulator with the scalar alpha: ties go to even,
    and the all-zero rule is applied to the scaled slice."""
    g = golden("inf_controls")
    hs, il, d = T_(g["lr_hs"]), T_(g["lr_ilens"]), T_(g["lr_d"])
    for i, a in enumerate(g["lr_alphas"].tolist()):
        out, used = P.length_regulator(hs, d, il, torch.full(d.shape, a))
        assert torch.equal(out, T_(g[f"lr_out{i}"])), a
        assert torch.equal(used.sum(1).max(), torch.tensor(out.shape[1]))
    _, used = P.length_regulator(hs, d, il, torch.full(d.shape, 0.4))
    assert torch.equal(used[1, :5], torch.ones(5, dtype=torch.int64))       # every 1 * 0.4 rounds to 0 -> all ones


@pytest.fixture(scope="module")
def model(weights):
    m = FeedForwardTransformer(68, 80, load_hp())
    m.load_state_dict(weights, strict=True)
    return m.eval()


def batch():
    xs = torch.zeros(3, 12, dtype=torch.int64)
    xs[:, :5] = 7
    return xs, torch.tensor([12, 4, 5])


@pytest.mark.parametrize("name", ["speed", "pitch", "energy"])
@pytest.mark.parametrize("bad", [0.0, -1.0, float("nan"), float("inf"), 1e-50, 1e39])
def test_invalid_factors_raise(model, name, bad):
    """Finite and > 0 after rounding to fp32 (1e-50 rounds to 0, 1e39 to inf), as a number, per utterance and per phoneme."""
    xs, il = batch()
    with pytest.raises(ValueError, match="finite and > 0"):
        model.synthesize(xs, il, **{name: bad})
    with pytest.raises(ValueError, match="finite and > 0"):
        model.synthesize(xs, il, **{name: torch.tensor([1.0, bad, 1.0], dtype=torch.float64)})
    per_phoneme = torch.ones(3, 12, dtype=torch.float64)
    per_phoneme[2, 4] = bad
    with pytest.raises(ValueError, match="finite and > 0"):
        model.synthesize(xs, il, **{name: per_phoneme})
    with pytest.raises(ValueError, match="finite and > 0"):
        model.inference_controlled(xs[0], **{name: bad})


def test_factors_past_ilens_are_ignored(model):
    """A bad value where no phoneme is gets through validation (and then fails on the CPU model, loudly)."""
    xs, il = batch()
    per_phoneme = torch.ones(3, 12)
    per_phoneme[1, 4:] = 0.0                    # ilens[1] == 4
    with pytest.raises(_lib.Fs2Error, match="no CPU fallback"):
        model.synthesize(xs, il, speed=per_phoneme)


@pytest.mark.parametrize("shape", [(4,), (3, 13), (3, 11), (1, 12), (3, 12, 1)])
def test_wrong_shapes_raise(model, shape):
    xs, il = batch()
    with pytest.raises(ValueError, match=r"must be a number"):
        model.synthesize(xs, il, pitch=torch.ones(shape))
    with pytest.raises(ValueError, match=r"must be a number or a \[T=12\]"):
        model.inference_controlled(xs[0], energy=torch.ones(shape))


def test_cpu_tensors_raise(model):
    xs, il = batch()
    with pytest.raises(_lib.Fs2Error, match="no CPU fallback"):
        model.synthesize(xs, il, speed=1.25, pitch=torch.ones(3), energy=torch.ones(3, 12))
    with pytest.raises(_lib.Fs2Error, match="no CPU fallback"):
        model.inference_controlled(xs[0], speed=torch.full((12,), 1.5))


def test_controls_rejected_without_reference_semantics(model):
    """Teacher-forced and reference-semantics batched calls have no defined behaviour for controls."""
    xs, il = batch()
    ctl = (torch.ones(3, 12), None, None)
    ol, ds, e = torch.full((3,), 24), torch.full((3, 12), 2), torch.zeros(3, 24)
    with pytest.raises(ValueError, match="inference only"):
        model._forward(xs, il, ol, ds, e, e, _controls=ctl)
    with pytest.raises(ValueError, match="inference only"):
        model._forward(xs, il, ol, ds, e, e, per_utterance=True, _controls=ctl)
    with pytest.raises(ValueError, match="per_utterance=True"):
        model._forward(xs, il, is_inference=True, _controls=ctl)


def test_library_exports_control_entry_points():
    lib = _lib.load()
    header = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    for name in ("fs2_length_plan_ex", "fs2_length_gather_ex", "fs2_decode_ctl"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES, name
        assert f"int {name}(" in header, name


def test_touched_kernels_do_not_spill():
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "*.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = "".join(open(r).read() for r in reports)
    for kernel in ("length_plan_kernel", "length_gather_kernel", "row_norm_kernel"):
        props = re.findall(r"Function properties for \S*%s\S*\n(.*)" % kernel, text)
        assert props, kernel
        for line in props:
            assert "0 bytes spill stores, 0 bytes spill loads" in line, (kernel, line)
