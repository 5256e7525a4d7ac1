"""iSTFTNet vocoder without a GPU: the key list of tests/golden/istftnet_state_dict_keys.json against both module trees
(ISTFTNetVocoder and oracle/istftnet_oracle.py), the config refusals in Python and in C, config forms and config.json
discovery, checkpoint loading in every form, the launch and FLOP counts, the head's per-sample index form
(tests/_istftnet_head.py) against the oracle's torch.istft path, the window plan against the float64 oracle's NaN cone,
the C entry points and the ptxas report of csrc/istftnet.cu."""
import ctypes as C
import glob
import json
import os
import re

import pytest
import torch

import _istftnet_head as H
from conftest import GOLDEN, REPO
from fastspeech2_b200 import _lib
from fastspeech2_b200.hifigan import CONFIGS as HCONFIGS
from fastspeech2_b200.istftnet import CONFIGS, ISTFTNetVocoder, check_config, load_config
from oracle import istftnet_oracle as O


def _golden():
    return [(k, tuple(s)) for k, s in json.load(open(os.path.join(GOLDEN, "istftnet_state_dict_keys.json")))["v1"]]


def _perturbed(g, seed):
    torch.manual_seed(seed)
    with torch.no_grad():
        for n, p in g.named_parameters():
            if n.endswith("weight_g"):
                p.mul_(torch.rand(p.shape) + 0.5)
    return g.eval()


def test_key_list_matches_both_module_trees():
    want = _golden()
    assert len(want) == 120 and ("conv_post.weight_v", (18, 128, 7)) in want and ("conv_post.bias", (18,)) in want
    assert [(k, tuple(v.shape)) for k, v in O.Generator(CONFIGS["v1"]).state_dict().items()] == want
    assert [(k, tuple(v.shape)) for k, v in ISTFTNetVocoder("v1").state_dict().items()] == want
    assert sum(p.numel() for p in ISTFTNetVocoder("v1").parameters()) == 13262244


def test_launches_and_flops_against_hand_counts():
    v = ISTFTNetVocoder("v1")
    assert v.launches() == 4 + 2 * (2 + 3 * 12 + 1) == 82
    # conv_pre 80*512*7; ups 512*256*16 and 8*256*128*16; MRFs 8 * 6*256^2*(3+7+11) and 64 * 6*128^2*21; conv_post 64*128*18*7
    hand = 80 * 512 * 7 + 512 * 256 * 16 + 8 * 6 * 256 ** 2 * 21 + 8 * 256 * 128 * 16 + 64 * 6 * 128 ** 2 * 21 + 64 * 128 * 18 * 7
    assert v.flops_per_frame() == 2 * hand == 411582464


def test_config_forms_and_refusals():
    assert load_config("v1") == load_config(dict(CONFIGS["v1"], batch_size=16)) == load_config("V1")
    with pytest.raises(ValueError, match="gen_istft_n_fft"):
        ISTFTNetVocoder(HCONFIGS["v1"])                                 # a hifi-gan config
    with pytest.raises(ValueError, match="gen_istft_hop_size"):
        ISTFTNetVocoder({k: v for k, v in CONFIGS["v1"].items() if k != "gen_istft_hop_size"})
    for edits, what in ((dict(gen_istft_n_fft=15), "gen_istft_n_fft"), (dict(gen_istft_n_fft=32, gen_istft_hop_size=8), "gen_istft_n_fft"),
                        (dict(gen_istft_n_fft=16, gen_istft_hop_size=16), "gen_istft_hop_size"),
                        (dict(gen_istft_n_fft=12, gen_istft_hop_size=5), "gen_istft_hop_size"),
                        (dict(gen_istft_hop_size=2), "product"), (dict(upsample_rates=[8, 4], upsample_kernel_sizes=[16, 8]), "product"),
                        (dict(upsample_kernel_sizes=[16, 15]), "upsample_kernel_sizes"), (dict(upsample_initial_channel=96), "upsample_initial_channel"),
                        (dict(resblock="3"), "resblock"), (dict(resblock_kernel_sizes=[3, 7, 10]), "resblock_kernel_sizes"),
                        (dict(num_mels=100), "num_mels"), (dict(gen_istft_n_fft=16.0), "gen_istft_n_fft")):
        with pytest.raises(ValueError, match=what):
            check_config(load_config(dict(CONFIGS["v1"], **edits)))
    # other accepted forms: n_fft 8 with hop 2 behind rates [8, 8, 2]
    check_config(load_config(dict(CONFIGS["v1"], upsample_rates=[8, 8, 2], upsample_kernel_sizes=[16, 16, 4], gen_istft_n_fft=8,
                                  gen_istft_hop_size=2)))


def test_create_validates_the_config_in_c():
    """fs2_istftnet_create refuses what check_config refuses, before it touches the device, naming the field."""
    lib = _lib.load()
    base = ISTFTNetVocoder("v1")

    def create(**edits):
        c = base._c_config()
        for k, v in edits.items():
            if k == "rate":
                c.gen.upsample_rates[0] = v
            elif k == "kernel":
                c.gen.upsample_kernel_sizes[0] = v
            elif k in ("istft_n_fft", "istft_hop"):
                setattr(c, k, v)
            else:
                setattr(c.gen, k, v)
        h = C.c_void_p()
        return lib.fs2_istftnet_create(C.byref(h), _lib.MATH_3XTF32, C.byref(c))

    for edits, what in ((dict(istft_hop=2), b"istft_hop (2)"), (dict(rate=4, kernel=8), b"product"), (dict(istft_n_fft=15), b"istft_n_fft"),
                        (dict(istft_n_fft=32, istft_hop=8), b"istft_n_fft = 32 is above 16"), (dict(istft_hop=16), b"istft_hop"),
                        (dict(istft_hop=3), b"istft_hop"), (dict(istft_hop=0), b"istft_hop"), (dict(resblock=3), b"resblock"),
                        (dict(kernel=15), b"upsample_kernel_sizes"), (dict(upsample_initial_channel=96), b"upsample_initial_channel"),
                        (dict(num_dilations=2), b"num_dilations")):
        assert create(**edits) == -1, edits
        err = lib.fs2_last_error()
        assert what in err and err.startswith(b"fs2_istftnet_create"), (edits, err)
    # the HiFi-GAN entry keeps its own product rule and message
    h = C.c_void_p()
    assert lib.fs2_hifigan_create(C.byref(h), _lib.MATH_3XTF32, C.byref(base._c_config().gen)) == -1
    assert b"fs2_hifigan_create: the product of upsample_rates is 64, not the hop 256" in lib.fs2_last_error()


def test_config_json_discovery_and_checkpoint_forms(tmp_path):
    g = _perturbed(O.Generator(CONFIGS["v1"]), 0)
    sd = g.state_dict()
    path = tmp_path / "g_00100000"
    torch.save({"generator": sd}, path)
    with pytest.raises(ValueError, match="config.json"):
        ISTFTNetVocoder.from_checkpoint(str(path))
    (tmp_path / "config.json").write_text(json.dumps(dict(CONFIGS["v1"], batch_size=16, sampling_rate=22050)))
    want = {k: v.float() for k, v in ISTFTNetVocoder.from_checkpoint(str(path)).state_dict().items()}
    assert all(torch.equal(want[k], v) for k, v in sd.items())
    bare = ISTFTNetVocoder.from_checkpoint(dict(sd), config="v1")
    assert all(torch.equal(bare.state_dict()[k], v) for k, v in sd.items())
    with pytest.raises(ValueError, match="config is required"):
        ISTFTNetVocoder.from_checkpoint(dict(sd))
    g.remove_weight_norm()
    plain = ISTFTNetVocoder.from_checkpoint({"generator": g.state_dict()}, config="v1")
    for m, n in ((plain.conv_post, "conv_post"), (plain.ups[1], "ups.1")):
        assert torch.equal(m.folded(), g.state_dict()[f"{n}.weight"]), n
    bad = dict(sd)
    bad["conv_post.weight_v"] = torch.zeros(1, 128, 7)                  # a hifi-gan conv_post
    with pytest.raises(ValueError, match="conv_post.weight_v"):
        ISTFTNetVocoder.from_checkpoint(bad, config="v1")


@pytest.mark.parametrize("frames", [1, 2, 3, 7, 16, 40])
def test_head_index_form_matches_the_oracle_istft(frames):
    """tests/_istftnet_head.py (reflect, conv taps, c2r sum, overlap-add and envelope per output sample) against the
    oracle's ReflectionPad1d + conv_post + torch.istft on utterances of 1 to 40 frames (64 last-level rows each)."""
    torch.manual_seed(frames)
    g = O.Generator(dict(CONFIGS["v1"], upsample_initial_channel=128)).double().eval()     # C_U = 32
    T = 64 * frames
    x = torch.randn(1, 32, T, dtype=torch.float64)
    with torch.no_grad():
        want = g.head(x)[0].numpy()
        w, b = g.conv_post.weight.numpy(), g.conv_post.bias.numpy()
    got = H.head(x[0].T.numpy(), w, b, g.n_fft, g.hop)
    assert got.shape == want.shape == (4 * T,)
    assert abs(got - want).max() <= 1e-12 * abs(want).max()


def test_head_reach_is_derived_from_the_index_form():
    """Audio samples [256 c0, 256 c1) read last-level rows [64 c0 - 5, 64 c1 + 3]: a reach of 5 for n_fft 16, hop 4."""
    assert ISTFTNetVocoder("v1").head_reach() == H.reach(16, 4) == 5
    for n, hop in ((8, 2), (4, 1), (16, 8), (12, 4)):
        cfg = dict(CONFIGS["v1"], gen_istft_n_fft=n, gen_istft_hop_size=hop)
        assert 4 + (n // 2 - 1) // hop == H.reach(n, hop), (n, hop)
        if 256 % hop == 0 and hop in (2, 4, 8):
            rates = {2: [8, 8, 2], 4: [8, 8], 8: [8, 4]}[hop]
            cfg.update(upsample_rates=rates, upsample_kernel_sizes=[2 * u for u in rates])
            assert ISTFTNetVocoder(cfg).head_reach() == H.reach(n, hop)
    plan = ISTFTNetVocoder("v1").window_plan()
    assert plan == {"reach": [10, 9], "halo": [13, 80, 72], "R": 60}


def test_head_reach_matches_the_nan_cone_of_the_head():
    """A NaN in last-level row 64 c0 - 5 reaches the samples of rows [64 c0, 64 c1); one in row 64 c0 - 6 does not; on the
    right, rows 64 c1 + 3 and 64 c1 + 4."""
    g = O.Generator(dict(CONFIGS["v1"], upsample_initial_channel=128)).double().eval()
    T, r0, r1 = 64 * 6, 128, 192
    x = torch.randn(1, 32, T, dtype=torch.float64)

    def reaches(row):
        xx = x.clone()
        xx[0, :, row] = float("nan")
        with torch.no_grad():
            return bool(torch.isnan(g.head(xx)[0, 4 * r0: 4 * r1]).any())
    assert reaches(r0 - 5) and not reaches(r0 - 6)
    assert reaches(r1 + 3) and not reaches(r1 + 4)


def test_plan_reach_matches_the_nan_cone():
    """A NaN at mel frame c0 - h_0 reaches the audio of the window [c0, c1), one at c0 - h_0 - 1 does not, and the same on
    the right: the float64 oracle at reduced widths."""
    h0 = ISTFTNetVocoder("v1").window_plan()["halo"][0]
    g = _perturbed(O.Generator(dict(CONFIGS["v1"], upsample_initial_channel=64)), 4).double()
    c0, nf = h0 + 2, 3
    c1, n = c0 + nf, c0 + nf + h0 + 2
    mel = torch.randn(1, 80, n, dtype=torch.float64) - 5

    def reaches(frame):
        m = mel.clone()
        m[0, :, frame] = float("nan")
        with torch.no_grad():
            return bool(torch.isnan(g(m)[0, 0, c0 * 256: c1 * 256]).any())
    assert reaches(c0 - h0) and not reaches(c0 - h0 - 1)
    assert reaches(c1 - 1 + h0) and not reaches(c1 + h0)


def test_window_rows_and_size_checks():
    v = ISTFTNetVocoder("v1", math_mode="fp32")
    assert v._window_rows(4, 32) == (4 * (64 * 32 + 144), "B * (64 * n_frames + 144)")
    assert v._rows(2, 100) == (2 * 100 * 64, "B * Lmax * 64", "row")
    with pytest.raises(ValueError, match="65535"):
        v._check_size(64, 3000)


def test_library_exports_istftnet_entry_points():
    lib = _lib.load()
    header = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    for name in ("fs2_istftnet_create", "fs2_istftnet_load", "fs2_istftnet_workspace_bytes", "fs2_istftnet",
                 "fs2_istftnet_window_workspace_bytes", "fs2_istftnet_window", "fs2_op_istftnet_head"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES, name
        assert f"int {name}(" in header, name
    assert hasattr(lib, "fs2_istftnet_destroy") and "void fs2_istftnet_destroy(" in header
    for k in ("BAD_LENGTH", "RANGE", "BAD_START"):
        assert int(re.search(rf"#define FS2_ISTFTNET_{k} (\d+)", header).group(1)) == getattr(_lib, f"FS2_ISTFTNET_{k}")


def test_head_op_rejects_bad_arguments_on_the_host():
    lib = _lib.load()
    p = 256

    def head(C_=128, n=16, hop=4, x=p, B=2, Lp=40):
        return lib.fs2_op_istftnet_head(C_, n, hop, x, p, B, Lp, p, p, p, None)
    for kw, what in ((dict(C_=48), b"C must"), (dict(n=18), b"n_fft"), (dict(n=15), b"n_fft"), (dict(hop=16), b"hop"),
                     (dict(hop=3), b"hop"), (dict(x=None), b"null"), (dict(x=p + 4), b"aligned"), (dict(B=0), b"shape")):
        assert head(**kw) == -1, kw
        assert what in lib.fs2_last_error(), (kw, lib.fs2_last_error())


def test_head_kernel_does_not_spill():
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "istftnet.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = open(reports[0]).read()
    props = re.findall(r"Function properties for (\S+)\n(.*)", text)
    assert [n for n, _ in props if "istftnet_head_kernel" in n] and len(props) == 1, props
    assert "0 bytes spill stores, 0 bytes spill loads" in props[0][1], props
