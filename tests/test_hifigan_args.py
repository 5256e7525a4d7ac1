"""HiFi-GAN vocoder without a GPU: the key lists of tests/golden/hifigan_state_dict_keys.json against both module trees
(HiFiGANVocoder and oracle/hifigan_oracle.py), the config refusals, config.json discovery, checkpoint loading in every
form, the size limits, the C entry points' host-side checks and the ptxas report of csrc/hifigan.cu."""
import glob
import json
import os
import re

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from conftest import GOLDEN, REPO
from fastspeech2_b200 import _lib
from fastspeech2_b200.hifigan import CONFIGS, HiFiGANVocoder, add_layers, check_config, load_config
from oracle import hifigan_oracle as O


def _golden(name):
    return [(k, tuple(s)) for k, s in json.load(open(os.path.join(GOLDEN, "hifigan_state_dict_keys.json")))[name]]


def _oracle(name, seed=0):
    torch.manual_seed(seed)
    g = O.Generator(CONFIGS[name])
    with torch.no_grad():                      # move g away from |v| so that the fold is not the identity
        for n, p in g.named_parameters():
            if n.endswith("weight_g"):
                p.mul_(torch.rand(p.shape) + 0.5)
    return g.eval()


@pytest.mark.parametrize("name,n_keys", [("v1", 234), ("v2", 234), ("v3", 69)])
def test_key_lists_match_both_module_trees(name, n_keys):
    want = _golden(name)
    assert len(want) == n_keys
    assert [(k, tuple(v.shape)) for k, v in O.Generator(CONFIGS[name]).state_dict().items()] == want
    tree = add_layers(nn.Module(), load_config(name))
    assert [(k, tuple(v.shape)) for k, v in tree.state_dict().items()] == want
    if name != "v2":
        assert [(k, tuple(v.shape)) for k, v in HiFiGANVocoder(name).state_dict().items()] == want


def test_parameter_counts():
    counts = {n: sum(p.numel() for p in add_layers(nn.Module(), load_config(n)).parameters()) for n in CONFIGS}
    print(f"\nhifigan parameters: {counts}")
    assert counts == {"v1": 13936130, "v2": 928514, "v3": 1464322}
    assert counts["v1"] == sum(p.numel() for p in O.Generator(CONFIGS["v1"]).parameters())


def test_flops_and_launches_per_config():
    v1, v3 = HiFiGANVocoder("v1"), HiFiGANVocoder("v3")
    assert abs(v1.flops_per_frame() / 0.61e9 - 1) < 0.01 and abs(v3.flops_per_frame() / 45e6 - 1) < 0.01
    assert (v1.launches(), v3.launches()) == (160, 49)


def test_transposed_conv_g_is_per_input_channel():
    v = HiFiGANVocoder("v3")
    for i, (cin, cout) in enumerate(((256, 128), (128, 64), (64, 32))):
        assert tuple(v.state_dict()[f"ups.{i}.weight_g"].shape) == (cin, 1, 1)
        assert tuple(v.state_dict()[f"ups.{i}.bias"].shape) == (cout,)


def _folded_forward(v: HiFiGANVocoder, mel):
    """The generator in torch.nn.functional from HiFiGANVocoder's folded weights (what fs2_hifigan_load receives)."""
    cfg = v.config
    conv = lambda m, x, d=1: F.conv1d(x, m.folded(), m.bias.detach(), dilation=d, padding=d * (m.weight_v.shape[2] - 1) // 2)
    x = conv(v.conv_pre, mel)
    nk = len(cfg["resblock_kernel_sizes"])
    for i, u in enumerate(cfg["upsample_rates"]):
        x = F.conv_transpose1d(F.leaky_relu(x, 0.1), v.ups[i].folded(), v.ups[i].bias.detach(), stride=u, padding=u // 2)
        xs = None
        for j in range(nk):
            rb, dil, y = v.resblocks[i * nk + j], cfg["resblock_dilation_sizes"][j], x
            if cfg["resblock"] == "1":
                for c1, c2, d in zip(rb.convs1, rb.convs2, dil):
                    y = conv(c2, F.leaky_relu(conv(c1, F.leaky_relu(y, 0.1), d), 0.1)) + y
            else:
                for c, d in zip(rb.convs, dil):
                    y = conv(c, F.leaky_relu(y, 0.1), d) + y
            xs = y if xs is None else xs + y
        x = xs / nk
    return torch.tanh(conv(v.conv_post, F.leaky_relu(x)))


@pytest.mark.parametrize("name", ["v1", "v3"])
def test_folded_forward_equals_the_weight_norm_module(name):
    g = _oracle(name, 1)
    v = HiFiGANVocoder(name)
    v.load_state_dict(g.state_dict())
    mel = torch.randn(1, 80, 6) * 2 - 6
    with torch.no_grad():
        want = g(mel)
        got = _folded_forward(v, mel)
    assert got.shape == want.shape == (1, 1, 6 * 256)
    assert float((got - want).abs().max()) <= 1e-5                 # fp32 noise: the oneDNN kernels sum in other orders


def test_oracle_batched_is_per_utterance():
    g = _oracle("v3", 2)
    mels = torch.randn(2, 7, 80) * 2 - 6
    with torch.no_grad():
        audio = O.batched(g, mels, [7, 3])
        one = g(mels[1, :3].T[None])[0, 0]
    assert audio.shape == (2, 7 * 256) and torch.all(audio[1, 3 * 256:] == 0)
    assert torch.equal(audio[1, : 3 * 256], one)


def _with(name, **edits):
    cfg = json.loads(json.dumps(CONFIGS[name]))
    cfg.update(edits)
    return cfg


@pytest.mark.parametrize("cfg,field", [
    (_with("v1", upsample_rates=[8, 8, 2, 4], upsample_kernel_sizes=[16, 16, 4, 8]), "upsample_rates"),
    (_with("v1", upsample_rates=[8, 4, 4, 2], upsample_kernel_sizes=[16, 8, 8, 4]), None),
    (_with("v1", upsample_kernel_sizes=[16, 16, 4, 5]), "upsample_kernel_sizes"),
    (_with("v1", upsample_kernel_sizes=[16, 15, 4, 4]), "upsample_kernel_sizes"),
    (_with("v1", upsample_rates=[8, 8, 1, 4], upsample_kernel_sizes=[16, 16, 2, 8]), "upsample_rates"),
    (_with("v1", upsample_rates=[16, 16], upsample_kernel_sizes=[32, 32]), None),
    (_with("v1", upsample_rates=[256 // 3, 3], upsample_kernel_sizes=[170, 6]), "upsample_rates"),
    (_with("v1", num_mels=128), "num_mels"),
    (_with("v1", resblock="3"), "resblock"),
    (_with("v1", resblock=2), None),                                  # ResBlock2 uses the first two dilations
    (CONFIGS["v2"], "upsample_initial_channel"),
    (_with("v3", upsample_initial_channel=192), "upsample_initial_channel"),
    (_with("v3", upsample_initial_channel=4096), "upsample_initial_channel"),
    (_with("v1", resblock_kernel_sizes=[3, 6, 11]), "resblock_kernel_sizes"),
    (_with("v3", resblock_dilation_sizes=[[1], [2, 6], [3, 12]]), "resblock_dilation_sizes"),
])
def test_config_refusals_name_their_field(cfg, field):
    if field is None:
        check_config(load_config(cfg))
        return
    with pytest.raises(ValueError, match=field):
        HiFiGANVocoder(cfg)


def test_config_forms_and_missing_fields(tmp_path):
    path = tmp_path / "config.json"
    path.write_text(json.dumps(dict(CONFIGS["v3"], batch_size=16, sampling_rate=22050)))
    assert HiFiGANVocoder(str(path)).config == HiFiGANVocoder("v3").config == HiFiGANVocoder(CONFIGS["v3"]).config
    cfg = dict(CONFIGS["v1"])
    del cfg["resblock_dilation_sizes"]
    with pytest.raises(ValueError, match="resblock_dilation_sizes"):
        HiFiGANVocoder(cfg)
    with pytest.raises(ValueError, match="config"):
        HiFiGANVocoder(42)
    with pytest.raises(ValueError, match="math_mode"):
        HiFiGANVocoder("v3", math_mode="bf16")


def _plain(g):
    g2 = O.Generator(CONFIGS["v3"])
    g2.load_state_dict(g.state_dict())
    g2.remove_weight_norm()
    return g2


def test_from_checkpoint_forms_and_config_discovery(tmp_path):
    g = _oracle("v3", 3)
    sd = g.state_dict()
    d = tmp_path / "run"
    d.mkdir()
    path = d / "g_02500000"
    torch.save({"generator": sd}, path)
    with pytest.raises(ValueError, match="config"):
        HiFiGANVocoder.from_checkpoint(str(path))                    # no config.json yet
    with pytest.raises(ValueError, match="config"):
        HiFiGANVocoder.from_checkpoint({"generator": sd})
    (d / "config.json").write_text(json.dumps(CONFIGS["v3"]))
    for src, cfg in ((str(path), None), (path, None), ({"generator": sd}, "v3"), (sd, "v3"), (str(path), CONFIGS["v3"])):
        v = HiFiGANVocoder.from_checkpoint(src, config=cfg)
        assert v.config == HiFiGANVocoder("v3").config
        assert all(torch.equal(v.state_dict()[k], sd[k]) for k in sd)
    plain = _plain(g).state_dict()
    assert any(k.endswith(".weight") for k in plain) and not any(k.endswith("weight_g") for k in plain)
    v = HiFiGANVocoder.from_checkpoint({"generator": plain}, config="v3")
    for name, m in v.named_modules():
        if hasattr(m, "folded"):
            assert torch.equal(m.folded(), plain[f"{name}.weight"]), name
    with pytest.raises(ValueError, match="shape"):                   # a V3 file read with V1's config
        HiFiGANVocoder.from_checkpoint(sd, config="v1")


@pytest.mark.parametrize("edit,match", [
    (lambda sd: sd.pop("resblocks.4.convs.1.weight_v"), "missing key resblocks.4.convs.1.weight_v"),
    (lambda sd: sd.__setitem__("resblocks.9.convs.0.bias", torch.zeros(3)), "unexpected key resblocks.9.convs.0.bias"),
    (lambda sd: sd.__setitem__("ups.0.weight_g", torch.ones(128, 1, 1)), r"ups.0.weight_g has shape \(128, 1, 1\)"),
    (lambda sd: sd.__setitem__("conv_post.bias", torch.zeros(2)), "conv_post.bias has shape"),
])
def test_from_checkpoint_rejects_bad_keys_by_name(edit, match):
    sd = dict(O.Generator(CONFIGS["v3"]).state_dict())
    edit(sd)
    with pytest.raises(ValueError, match=match):
        HiFiGANVocoder.from_checkpoint({"generator": sd}, config="v3")


@pytest.fixture(scope="module")
def voc():
    return HiFiGANVocoder("v3")


@pytest.mark.parametrize("shape,olens,match", [
    ((2, 10), [10, 9], "mels"), ((2, 10, 40), [10, 9], "mels"), ((0, 10, 80), [], "mels"), ((2, 10, 80), [10], "olens"),
    ((2, 10, 80), [10.0, 9.0], "integer"), ((2, 10, 80), [10, 9], "CUDA")])
def test_bad_inputs_raise(voc, shape, olens, match):
    with pytest.raises(ValueError, match=match):
        voc(torch.zeros(shape), torch.tensor(olens))


def test_size_limits_raise():
    v = HiFiGANVocoder("v3", math_mode="fp32")
    with pytest.raises(ValueError, match="fp32"):
        v._check_size(1, 65535 * 128 // 256 + 1)
    v._check_size(1, 65535 * 128 // 256)
    t = HiFiGANVocoder("v3", math_mode="tf32")
    t._check_size(1, 65535 * 128 // 256 + 1)
    with pytest.raises(ValueError, match="2\\^31"):
        t._check_size(64, (1 << 31) // (64 * 256))
    t._check_size(64, (1 << 31) // (64 * 256) - 1)


def test_library_exports_hifigan_entry_points():
    lib = _lib.load()
    header = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    for name in ("fs2_hifigan_create", "fs2_hifigan_load", "fs2_hifigan_workspace_bytes", "fs2_hifigan", "fs2_op_hifigan_resblock",
                 "fs2_op_hifigan_upsample"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES, name
        assert f"int {name}(" in header, name
    assert hasattr(lib, "fs2_hifigan_destroy") and "void fs2_hifigan_destroy(" in header
    assert int(re.search(r"#define FS2_HIFIGAN_MAX_UPSAMPLES (\d+)", header).group(1)) == _lib.FS2_HIFIGAN_MAX_UPSAMPLES
    assert int(re.search(r"#define FS2_HIFIGAN_MAX_KERNELS (\d+)", header).group(1)) == _lib.FS2_HIFIGAN_MAX_KERNELS


def test_create_validates_the_config_in_c():
    """fs2_hifigan_create refuses what check_config refuses, before it touches the device."""
    import ctypes as C
    lib = _lib.load()
    base = HiFiGANVocoder("v3")

    def create(**edits):
        c = base._c_config()
        for k, v in edits.items():
            if k == "rate":
                c.upsample_rates[0] = v
            elif k == "kernel":
                c.upsample_kernel_sizes[0] = v
            elif k == "rk":
                c.resblock_kernel_sizes[0] = v
            elif k == "dil":
                c.resblock_dilation_sizes[0][0] = v
            else:
                setattr(c, k, v)
        h = C.c_void_p()
        return lib.fs2_hifigan_create(C.byref(h), _lib.MATH_3XTF32, C.byref(c))

    for edits, what in ((dict(resblock=3), b"resblock"), (dict(rate=4, kernel=8), b"product"), (dict(kernel=15), b"upsample_kernel_sizes"),
                        (dict(rate=7, kernel=14), b"upsample_rates"), (dict(upsample_initial_channel=128), b"upsample_initial_channel"),
                        (dict(upsample_initial_channel=4096), b"upsample_initial_channel"), (dict(num_upsamples=0), b"num_upsamples"),
                        (dict(rk=4), b"resblock_kernel_sizes"), (dict(dil=0), b"resblock_dilation_sizes"),
                        (dict(num_dilations=3), b"num_dilations"), (dict(num_kernels=9), b"num_kernels")):
        assert create(**edits) == -1, edits
        assert what in lib.fs2_last_error(), (edits, lib.fs2_last_error())
    assert create(resblock=1, num_dilations=2) == -1


def test_single_layer_entries_reject_bad_arguments_on_the_host():
    """fs2_op_hifigan_resblock and fs2_op_hifigan_upsample refuse these before they touch memory (the pointers are never
    dereferenced)."""
    import ctypes as C
    lib = _lib.load()
    p = 256     # a stand-in non-null, aligned pointer
    wp = (C.c_void_p * 6)(*([p] * 6))

    def block(mode=_lib.MATH_3XTF32, type_=2, C_=64, k=3, dils=(1, 3), x=p, out=p, B=2, Lp=40):
        d = (C.c_int * len(dils))(*dils)
        return lib.fs2_op_hifigan_resblock(mode, type_, C_, k, len(dils), d, x, p, B, Lp, wp, wp, out, p, None)

    def upsample(mode=_lib.MATH_3XTF32, Cin=64, Cout=32, u=2, x=p, B=2, Lin=40):
        return lib.fs2_op_hifigan_upsample(mode, Cin, Cout, u, x, p, B, Lin, p, p, p, p, None)

    for mode in (-1, 4):
        assert block(mode=mode) == -1 and b"math_mode" in lib.fs2_last_error()
        assert upsample(mode=mode) == -1 and b"math_mode" in lib.fs2_last_error()
    assert block(type_=3) == -1 and b"type" in lib.fs2_last_error()
    for C_ in (0, 16, 48, 80):
        assert block(C_=C_) == -1 and b"C must be" in lib.fs2_last_error()
    for k in (0, 2, 33):
        assert block(k=k) == -1 and b"k must be" in lib.fs2_last_error()
    assert block(type_=1, dils=(1, 3)) == -1 and b"nd must be" in lib.fs2_last_error()
    assert block(dils=(0, 1)) == -1 and b"dilation" in lib.fs2_last_error()
    assert block(x=None) == -1 and b"null" in lib.fs2_last_error()
    assert block(x=p + 8) == -1 and b"aligned" in lib.fs2_last_error()
    assert block(out=p + 16) == -1 and b"aligned" in lib.fs2_last_error()
    assert block(B=0) == -1 and b"shape" in lib.fs2_last_error()
    assert block(mode=_lib.MATH_FP32, B=65535, Lp=129) == -1 and b"too many rows" in lib.fs2_last_error()
    for u in (0, 1, 3, 7):
        assert upsample(u=u) == -1 and b"rate" in lib.fs2_last_error()
    for Cin, Cout in ((40, 32), (64, 16), (0, 32)):
        assert upsample(Cin=Cin, Cout=Cout) == -1 and b"multiples of 32" in lib.fs2_last_error()
    assert upsample(x=None) == -1 and b"null" in lib.fs2_last_error()
    assert upsample(x=p + 4) == -1 and b"aligned" in lib.fs2_last_error()
    assert upsample(Lin=0) == -1 and b"shape" in lib.fs2_last_error()


def test_hifigan_kernels_do_not_spill():
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "hifigan.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = open(reports[0]).read()
    # instantiations: add, post (1 each), the rows producer (3 operand kinds x lrelu or none: HiFi-GAN's, iSTFTNet's and
    # BigVGAN's mel operand, upsampling operands and lrelu before the block convolutions)
    expected = {"hifigan_add_kernel": 1, "hifigan_post_kernel": 1, "hifigan_act_kernel": 6}
    for kernel, n in expected.items():
        props = re.findall(r"Function properties for \S*%s\S*\n(.*)" % kernel, text)
        assert len(props) == n, (kernel, len(props))
        for line in props:
            assert "0 bytes spill stores, 0 bytes spill loads" in line, (kernel, line)
    assert len(re.findall(r"Function properties for ", text)) == sum(expected.values())
