"""Host-side logic that needs no GPU: checkpoint layout, hp validation, loud failures,
and that the C-ABI library loads and exports every symbol include/fs2_b200.h declares."""
import ctypes
import json
import os
import re
import shutil
import subprocess

import pytest
import torch

from conftest import GOLDEN, REPO
from fastspeech2_b200 import FeedForwardTransformer, _lib
from fastspeech2_b200.hparams import load_hp


@pytest.fixture(scope="module")
def model():
    torch.manual_seed(0)
    return FeedForwardTransformer(68, 80, load_hp())


def test_state_dict_layout_matches_reference(model):
    ref = json.load(open(os.path.join(GOLDEN, "state_dict_keys.json")))
    sd = model.state_dict()
    assert list(sd.keys()) == [k for k, _, _ in ref]
    for k, shape, dtype in ref:
        assert list(sd[k].shape) == shape and str(sd[k].dtype) == dtype, k


def test_load_state_dict_strict(model, weights):
    missing = model.load_state_dict(weights, strict=True)
    assert not missing.missing_keys and not missing.unexpected_keys
    assert torch.equal(model.state_dict()["decoder.embed.4.pe"], weights["decoder.embed.4.pe"])


def test_fresh_init_matches_reference_conventions(model):
    m = FeedForwardTransformer(68, 80, load_hp())
    assert float(m.encoder.embed[-1].alpha) == 1.0 and float(m.decoder.embed[-1].alpha) == 1.0
    assert torch.count_nonzero(m.encoder.embed[0].weight[0]) == 0          # padding_idx = 0
    assert sum(p.numel() for p in m.parameters()) == 34015605              # BASELINE.md section 1


def test_cpu_inputs_fail_loudly(model):
    model.eval()
    x = torch.ones(2, 5, dtype=torch.int64)
    with pytest.raises(_lib.Fs2Error, match="no CPU fallback"):
        model._forward(x, torch.tensor([5, 5]), is_inference=True)


def test_train_mode_fails_loudly(model):
    model.train()
    with pytest.raises(NotImplementedError, match="eval"):
        model._forward(torch.ones(1, 5, dtype=torch.int64), torch.tensor([5]), is_inference=True)
    model.eval()


def test_unsupported_hp_is_rejected():
    hp = load_hp()
    hp.model.positionwise_layer_type = "linear"
    with pytest.raises(NotImplementedError):
        FeedForwardTransformer(68, 80, hp)
    hp = load_hp()
    hp.model.encoder_normalize_before = True
    with pytest.raises(NotImplementedError):
        FeedForwardTransformer(68, 80, hp)


def test_from_reference_checkpoint(tmp_path, weights):
    """The checkpoint layout train_fastspeech.py:235-244 writes, hp restored from its hp_str like inference.py:148-152."""
    from fastspeech2_b200.hparams import DEFAULT_YAML
    ck = {"model": weights, "optim": {"state": {}, "param_groups": []}, "step": 123000, "hp_str": open(DEFAULT_YAML).read(),
          "githash": "abc1234"}
    path = tmp_path / "fs2_abc1234_123k_steps.pyt"
    torch.save(ck, path)
    m = FeedForwardTransformer.from_checkpoint(str(path))
    assert not m.training and m.idim == 68 and m.odim == 80
    got = m.state_dict()
    assert list(got.keys()) == list(weights.keys())
    assert all(torch.equal(got[k], weights[k]) for k in weights)
    old_style = FeedForwardTransformer.from_checkpoint(dict(weights), hp=load_hp())       # bare state_dict (--old_model)
    assert torch.equal(old_style.state_dict()["feat_out.weight"], weights["feat_out.weight"])
    with pytest.raises(ValueError):
        FeedForwardTransformer.from_checkpoint(dict(weights))


def test_precision_names(model):
    """The extra `precision` keyword: default from FS2_PRECISION else "3xf16" (the reference-precision mode); unknown names are rejected; the header's
    FS2_MATH_* values and the ctypes table agree."""
    assert model.precision == os.environ.get("FS2_PRECISION", "3xf16")
    with pytest.raises(ValueError):
        FeedForwardTransformer(68, 80, load_hp(), precision="bf16")
    hdr = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    macros = {k: int(v) for k, v in re.findall(r"#define FS2_MATH_(\w+) (\d+)", hdr)}
    assert macros == {"FP32": _lib.MATH_MODES["fp32"], "TF32": _lib.MATH_MODES["tf32"], "3XTF32": _lib.MATH_MODES["3xtf32"],
                      "F16": _lib.MATH_MODES["f16"]}
    assert _lib.MATH_MODES["3xf16"] == _lib.MATH_MODES["3xtf32"]


def test_library_exports_every_declared_symbol():
    header = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    declared = set(re.findall(r"\b(fs2_[a-z0-9_]+)\s*\(", header))
    declared -= {"fs2_handle", "fs2_config", "fs2_weight_desc"}
    assert declared == set(_lib.ALL_SYMBOLS), declared ^ set(_lib.ALL_SYMBOLS)
    lib = ctypes.CDLL(_lib.LIB_PATH)   # loads without a GPU (cudart is linked statically)
    for name in declared:
        assert hasattr(lib, name), name
    lib.fs2_version.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.fs2_version()


def test_library_rejects_bad_arguments_without_a_gpu():
    lib = _lib.load()
    assert lib.fs2_length_gather(None, None, None, 1, 1, 256, None, 8, None) == -1
    assert b"null" in lib.fs2_last_error()


@pytest.mark.skipif(shutil.which("gcc") is None, reason="gcc not available")
def test_row_norm_desc_layout_matches_header(tmp_path):
    """_lib.RowNormDesc has fs2_row_norm_desc's fields in order, at the header's offsets and size; the row-kernel entries
    take as many arguments as the header declares."""
    header = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    fields = [n for n, _ in _lib.RowNormDesc._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "fs2_b200.h"\nint main(void) {\n'
                   + "".join(f'  printf("%zu ", offsetof(fs2_row_norm_desc, {n}));\n' for n in fields)
                   + '  printf("%zu\\n", sizeof(fs2_row_norm_desc));\n  return 0;\n}\n')
    exe = str(tmp_path / "layout")
    r = subprocess.run(["gcc", "-std=c99", "-I", os.path.join(REPO, "include"), str(src), "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    want = [getattr(_lib.RowNormDesc, n).offset for n in fields] + [ctypes.sizeof(_lib.RowNormDesc)]
    assert got == want
    body = re.search(r"typedef struct fs2_row_norm_desc \{(.*?)\} fs2_row_norm_desc;", header, re.S).group(1)
    assert re.findall(r"\**(\w+)\s*[;,]", body) == fields
    for name in ("fs2_op_row_norm", "fs2_op_variance_embed_add", "fs2_embed_posenc"):
        params = re.search(rf"int {name}\((.*?)\);", header, re.S).group(1)
        assert len(params.split(",")) == len(_lib.SIGNATURES[name]), name


def test_embed_posenc_binding_takes_both_forms():
    """The binding passes planes and lens as NULL when a caller omits them (the entry's form before they existed); either
    form reaches the library, which refuses the null xs before any launch."""
    lib = _lib.load()
    a = 0x10000
    assert lib.fs2_embed_posenc(None, a, 10, a, a, 2, 4, 256, a, None) == -1 and b"null" in lib.fs2_last_error()
    assert lib.fs2_embed_posenc(None, a, 10, a, a, 2, 4, 256, a, None, None, None) == -1 and b"null" in lib.fs2_last_error()
    with pytest.raises(TypeError):
        lib.fs2_embed_posenc(None, a, 10, a, a, 2, 4, 256, a, None, None)
