"""MelGAN vocoder without a GPU: the CPU oracle's size and keys against tests/golden/melgan_state_dict_keys.json, the
weight-norm fold, checkpoint loading in both key sets, the torch.hub hook of the drop-in launcher, argument validation,
the C entry points and the ptxas report of the new kernels."""
import glob
import json
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, REPO
from fastspeech2_b200 import _lib
from fastspeech2_b200 import dropin_run
from fastspeech2_b200.melgan import MelGANVocoder
from oracle import melgan_oracle as O


def _golden():
    return [(k, tuple(s)) for k, s in json.load(open(os.path.join(GOLDEN, "melgan_state_dict_keys.json")))]


def _oracle(seed=0):
    torch.manual_seed(seed)
    g = O.Generator()
    with torch.no_grad():                      # move g away from |v| so that the fold is not the identity
        for name, p in g.named_parameters():
            if name.endswith("weight_g"):
                p.mul_(torch.rand(p.shape) + 0.5)
    return g.eval()


def test_oracle_size_and_keys_match_the_golden_list():
    g = O.Generator()
    assert sum(p.numel() for p in g.parameters()) == 4266050
    assert [(k, tuple(v.shape)) for k, v in g.state_dict().items()] == _golden()
    assert len(_golden()) == 126


def test_vocoder_parameters_carry_the_same_keys():
    v = MelGANVocoder()
    assert [(k, tuple(t.shape)) for k, t in v.state_dict().items()] == _golden()
    assert sum(p.numel() for p in v.parameters()) == 4266050


def test_transposed_conv_g_is_per_input_channel():
    g, v = O.Generator(), MelGANVocoder()
    for i, (cin, cout) in zip((3, 6, 9, 12), ((512, 256), (256, 128), (128, 64), (64, 32))):
        assert tuple(g.state_dict()[f"generator.{i}.weight_g"].shape) == (cin, 1, 1)
        assert tuple(v.state_dict()[f"generator.{i}.weight_g"].shape) == (cin, 1, 1)
        assert tuple(v.state_dict()[f"generator.{i}.bias"].shape) == (cout,)


def _folded_forward(v: MelGANVocoder, mel):
    """The generator in torch.nn.functional from MelGANVocoder's folded weights (what fs2_melgan_load receives)."""
    gen = v.generator
    conv = lambda m, x, **kw: F.conv1d(x, m.folded(), m.bias.detach(), **kw)
    x = conv(gen[1], F.pad((mel + 5.0) / 5.0, (3, 3), mode="reflect"))
    for i in (3, 6, 9, 12):
        ct = gen[i]
        s = ct.weight_v.shape[2] // 2
        x = F.conv_transpose1d(F.leaky_relu(x, 0.2), ct.folded(), ct.bias.detach(), stride=s, padding=s // 2)
        for j, (blk, sc) in enumerate(zip(gen[i + 1].blocks, gen[i + 1].shortcuts)):
            d = 3 ** j
            h = conv(blk[2], F.pad(F.leaky_relu(x, 0.2), (d, d), mode="reflect"), dilation=d)
            x = conv(sc, x) + conv(blk[4], F.leaky_relu(h, 0.2))
    return torch.tanh(conv(gen[16], F.pad(F.leaky_relu(x, 0.2), (3, 3), mode="reflect")))


def test_folded_forward_equals_the_weight_norm_module():
    g = _oracle(1)
    v = MelGANVocoder()
    v.load_state_dict(g.state_dict())
    mel = torch.randn(1, 80, 24) * 2 - 6
    with torch.no_grad():
        want = g(mel)
        got = _folded_forward(v, mel)
    assert got.shape == want.shape == (1, 1, 24 * 256)
    assert float((got - want).abs().max()) <= 1e-5                 # fp32 noise: the oneDNN kernels sum in other orders


def test_oracle_batched_matches_inference():
    g = _oracle(2)
    mels = torch.randn(2, 9, 80) * 2 - 6
    with torch.no_grad():
        audio = O.batched(g, mels, [9, 4])
        i16 = g.inference(mels[1, :4].T[None])
    assert audio.shape == (2, 9 * 256) and torch.all(audio[1, 4 * 256:] == 0)
    assert torch.equal(MelGANVocoder.quantize(audio[1, : 4 * 256]), i16)


def _plain(g):
    g2 = O.Generator()
    g2.load_state_dict(g.state_dict())
    g2.eval(inference=True)                          # the hub object's remove_weight_norm
    return g2


def test_from_checkpoint_accepts_both_key_sets_and_the_wrapper(tmp_path):
    g = _oracle(3)
    sd = g.state_dict()
    plain = _plain(g).state_dict()
    assert any(k.endswith(".weight") for k in plain) and not any(k.endswith("weight_g") for k in plain)
    path = tmp_path / "melgan.pt"
    torch.save({"model_g": sd, "model_d": {}, "optim_g": {}, "optim_d": {}, "step": 7, "epoch": 1, "hp_str": "", "githash": "x"}, path)
    for src in (sd, {"model_g": sd}, str(path)):
        v = MelGANVocoder.from_checkpoint(src)
        assert all(torch.equal(v.state_dict()[k], sd[k]) for k in sd)
    # plain weights: v = w and g = |w| fold back to w bit for bit
    v = MelGANVocoder.from_checkpoint({"model_g": plain})
    for name, m in v.named_modules():
        if hasattr(m, "folded"):
            assert torch.equal(m.folded(), plain[f"{name}.weight"]), name


@pytest.mark.parametrize("edit,match", [
    (lambda sd: sd.pop("generator.7.blocks.1.4.weight_v"), "missing key generator.7.blocks.1.4.weight_v"),
    (lambda sd: sd.__setitem__("generator.99.bias", torch.zeros(3)), "unexpected key generator.99.bias"),
    (lambda sd: sd.__setitem__("generator.3.weight_g", torch.ones(256, 1, 1)), r"generator.3.weight_g has shape \(256, 1, 1\)"),
    (lambda sd: sd.__setitem__("generator.16.bias", torch.zeros(2)), "generator.16.bias has shape"),
])
def test_from_checkpoint_rejects_bad_keys_by_name(edit, match):
    sd = dict(O.Generator().state_dict())
    edit(sd)
    with pytest.raises(ValueError, match=match):
        MelGANVocoder.from_checkpoint({"model_g": sd})


def test_state_dict_round_trips():
    g = _oracle(4)
    v = MelGANVocoder()
    v.load_state_dict(g.state_dict())
    w = MelGANVocoder()
    w.load_state_dict(v.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(v.state_dict().values(), w.state_dict().values()))


@pytest.fixture
def fake_hub(monkeypatch):
    calls = []
    monkeypatch.setattr(torch.hub, "load", lambda repo, model, *a, **k: calls.append((repo, model)) or "original")
    return calls


def test_dropin_hook_serves_only_seungwonpark_melgan(tmp_path, fake_hub):
    path = tmp_path / "g.pt"
    torch.save({"model_g": O.Generator().state_dict()}, path)
    dropin_run.install_melgan_hub(str(path))
    assert isinstance(torch.hub.load("seungwonpark/melgan", "melgan"), MelGANVocoder)
    assert isinstance(torch.hub.load("seungwonpark/melgan:master", "melgan"), MelGANVocoder)
    assert torch.hub.load("seungwonpark/melgan", "other") == "original"
    assert torch.hub.load("NVIDIA/DeepLearningExamples:torchhub", "nvidia_waveglow") == "original"
    assert fake_hub == [("seungwonpark/melgan", "other"), ("NVIDIA/DeepLearningExamples:torchhub", "nvidia_waveglow")]


def test_dropin_launcher_installs_the_hook_from_the_environment(tmp_path):
    path = tmp_path / "g.pt"
    torch.save({"model_g": O.Generator().state_dict()}, path)
    script = tmp_path / "uses_hub.py"
    script.write_text("import torch\nv = torch.hub.load('seungwonpark/melgan', 'melgan')\nv.eval(inference=False)\n"
                      "print(type(v).__name__, len(v.state_dict()))\n")
    env = dict(os.environ, FS2_MELGAN_CHECKPOINT=str(path), PYTHONPATH=REPO)
    r = subprocess.run([sys.executable, "-m", "fastspeech2_b200.dropin_run", str(script)], cwd=str(tmp_path), env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert r.stdout.split() == ["MelGANVocoder", "126"]


@pytest.fixture(scope="module")
def voc():
    return MelGANVocoder()


@pytest.mark.parametrize("shape,olens,match", [
    ((2, 10), [10, 9], "mels"), ((2, 10, 40), [10, 9], "mels"), ((0, 10, 80), [], "mels"), ((2, 10, 80), [10], "olens"),
    ((2, 10, 80), [10.0, 9.0], "integer"), ((2, 10, 80), [10, 9], "CUDA")])
def test_bad_inputs_raise(voc, shape, olens, match):
    with pytest.raises(ValueError, match=match):
        voc(torch.zeros(shape), torch.tensor(olens))


def test_fp32_row_limit_raises_value_error():
    # fp32 runs its GEMMs on the CUDA-core family, whose grid puts 128-row tiles on grid.y (at most 65535)
    v = MelGANVocoder(math_mode="fp32")
    with pytest.raises(ValueError, match="fp32"):
        v._check_size(1, 65535 * 128 // 256)
    v._check_size(1, 65535 * 128 // 256 - 10)
    MelGANVocoder(math_mode="tf32")._check_size(1, 65535 * 128 // 256)


def test_bad_math_mode_and_inference_shape_raise(voc):
    with pytest.raises(ValueError, match="math_mode"):
        MelGANVocoder(math_mode="bf16")
    with pytest.raises(ValueError, match="mel"):
        voc.inference(torch.zeros(2, 80, 5))


def test_library_exports_melgan_entry_points():
    lib = _lib.load()
    header = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    for name in ("fs2_melgan_create", "fs2_melgan_load", "fs2_melgan_workspace_bytes", "fs2_melgan", "fs2_op_melgan_block",
                 "fs2_op_melgan_upsample"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES, name
        assert f"int {name}(" in header, name
    assert hasattr(lib, "fs2_melgan_destroy") and "void fs2_melgan_destroy(" in header


def test_single_layer_entries_reject_bad_arguments_on_the_host():
    """fs2_op_melgan_block and fs2_op_melgan_upsample refuse these before they touch memory (the pointers are never
    dereferenced)."""
    lib = _lib.load()
    p = 256     # a stand-in non-null, aligned pointer

    def block(mode=_lib.MATH_3XTF32, route=0, C=64, x=p, out=p, B=2, Lp=40, d=3):
        return lib.fs2_op_melgan_block(mode, route, C, x, p, B, Lp, d, p, p, p, p, p, p, out, p, None)

    def upsample(mode=_lib.MATH_3XTF32, Cin=64, Cout=32, s=2, x=p, B=2, Lin=40):
        return lib.fs2_op_melgan_upsample(mode, Cin, Cout, s, x, p, B, Lin, p, p, p, p, None)

    for mode in (-1, 4, 7):
        assert block(mode=mode) == -1 and b"math_mode" in lib.fs2_last_error()
        assert upsample(mode=mode) == -1 and b"math_mode" in lib.fs2_last_error()
    for route in (-1, 3):
        assert block(route=route) == -1 and b"route" in lib.fs2_last_error()
    for mode in (_lib.MATH_FP32, _lib.MATH_TF32):
        assert block(mode=mode, route=2) == -1 and b"fused route" in lib.fs2_last_error()
    for C in (0, 16, 48, 96, 512):
        assert block(C=C) == -1 and b"C must be" in lib.fs2_last_error()
    assert block(x=None) == -1 and b"null" in lib.fs2_last_error()
    assert block(x=p + 8) == -1 and b"aligned" in lib.fs2_last_error()
    assert block(out=p + 16) == -1 and b"aligned" in lib.fs2_last_error()
    assert block(d=0) == -1 and b"shape" in lib.fs2_last_error()
    assert block(B=0) == -1 and b"shape" in lib.fs2_last_error()
    assert block(mode=_lib.MATH_FP32, route=1, B=65535, Lp=129) == -1 and b"too many rows" in lib.fs2_last_error()
    for s in (0, 1, 3, 7):
        assert upsample(s=s) == -1 and b"stride" in lib.fs2_last_error()
    for Cin, Cout in ((40, 32), (64, 24), (0, 32)):
        assert upsample(Cin=Cin, Cout=Cout) == -1 and b"multiples of 16" in lib.fs2_last_error()
    assert upsample(x=None) == -1 and b"null" in lib.fs2_last_error()
    assert upsample(x=p + 4) == -1 and b"aligned" in lib.fs2_last_error()
    assert upsample(Lin=0) == -1 and b"shape" in lib.fs2_last_error()


def test_case_table_covers_the_block_instantiations():
    """The per-layer GPU cases (tests/test_gpu_melgan_kernels.py) reach every (C, precision) instantiation of the fused
    block on both routes, every dilation, and the geometry edges: empty, d + 1 and Lp utterances, a warp spanning two live
    utterances, a last CTA with a partial warp and an idle one; the upsampling lengths include 0, 1 and a tile tail."""
    import test_gpu_melgan_kernels as K
    assert K.check_coverage() == []
    assert sorted({(c.C, c.d) for c in K.BLOCK_CASES}) == [(C, d) for C in (32, 64, 128, 256) for d in (1, 3, 9)]
    assert [K.fused_blocks(m, C) for m in ("f16", "3xf16") for C in (32, 64, 128, 256)] == [True] * 3 + [False] + [True] * 2 + [False] * 2
    # 100 rows: only the warp at row 16 holds live rows of two utterances (0 and 1); the last CTA has 36 rows, 1 idle warp
    c = K.BlockCase(64, 1, 20, (20, 2, 0, 7, 20))
    assert K.straddles(c) == [16] and K.last_cta(c) == (36, 1)


def test_melgan_kernels_do_not_spill():
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "melgan.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = open(reports[0]).read()
    # instantiations: post (1), pre_operand and concat (3 operand kinds), taps (3 x 2), the fused residual block (4 channel
    # counts x f16 / 3xF16)
    expected = {"melgan_post_kernel": 1, "melgan_pre_operand_kernel": 3, "melgan_concat_kernel": 3, "melgan_taps_kernel": 6, "melgan_block_kernel": 8}
    for kernel, n in expected.items():
        props = re.findall(r"Function properties for \S*%s\S*\n(.*)" % kernel, text)
        assert len(props) == n, (kernel, len(props))
        for line in props:
            assert "0 bytes spill stores, 0 bytes spill loads" in line, (kernel, line)


def test_shared_weight_pack_kernels_do_not_spill():
    """The convolution weight pack, bias and zero-padding kernels MelGAN, HiFi-GAN and BigVGAN load their checkpoints
    through (csrc/vocoder_weights.cu)."""
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "vocoder_weights.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = open(reports[0]).read()
    for kernel in ("conv_pack_kernel", "conv_bias_kernel", "pad3_kernel"):
        props = re.findall(r"Function properties for \S*%s\S*\n(.*)" % kernel, text)
        assert len(props) == 1, (kernel, len(props))
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in props[0], (kernel, props[0])


def test_shared_window_prep_kernel_does_not_spill():
    """The one prep kernel MelGAN, HiFi-GAN and WaveGlow write their lengths and window descriptors with
    (csrc/vocoder_window.cu)."""
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "vocoder_window.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    props = re.findall(r"Function properties for (\S*)\n(.*)", open(reports[0]).read())
    assert len(props) == 1 and "ups_prep_kernel" in props[0][0], props
    assert "0 bytes spill stores, 0 bytes spill loads" in props[0][1], props[0]
