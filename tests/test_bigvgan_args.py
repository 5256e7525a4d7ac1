"""BigVGAN vocoder without a GPU: the key lists of tests/golden/bigvgan_state_dict_keys.json against both module trees
(BigVGANVocoder and oracle/bigvgan_oracle.py), the Activation1d index arithmetic the kernels use, the config refusals in
Python and in C, config.json discovery, checkpoint loading in every form, the window plan against a restatement and the
float64 oracle's NaN cone, the C entry points' host-side checks and the ptxas report of csrc/bigvgan.cu."""
import ctypes as C
import glob
import json
import os
import re

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import _bigvgan_window_plan as BP
from conftest import GOLDEN, REPO
from fastspeech2_b200 import _lib
from fastspeech2_b200.bigvgan import CONFIGS, BigVGANVocoder, add_layers, check_config, kaiser_sinc_filter1d, load_config
from oracle import bigvgan_oracle as O

NAMES = list(CONFIGS)
# reduced-width copies of the two topologies for the CPU oracle; the large one keeps a 24-wide stage
SMALL = {"base": dict(CONFIGS["base_22khz_80band"], upsample_initial_channel=128),
         "large": dict(CONFIGS["22khz_80band"], upsample_initial_channel=384)}


def _golden(name):
    return [(k, tuple(s)) for k, s in json.load(open(os.path.join(GOLDEN, "bigvgan_state_dict_keys.json")))[name]]


def _perturbed(g, seed):
    """g with every weight_g moved away from |v| and the Snake parameters away from their init."""
    torch.manual_seed(seed)
    with torch.no_grad():
        for n, p in g.named_parameters():
            if n.endswith("weight_g"):
                p.mul_(torch.rand(p.shape) + 0.5)
            elif n.endswith(".alpha") or n.endswith(".beta"):
                p.add_(torch.rand(p.shape) - 0.5)
    return g.eval()


@pytest.mark.parametrize("name,n_keys", [("base_22khz_80band", 526), ("22khz_80band", 784), ("v2_22khz_80band_fmax8k_256x", 783)])
def test_key_lists_match_both_module_trees(name, n_keys):
    want = _golden(name)
    assert len(want) == n_keys
    assert [(k, tuple(v.shape)) for k, v in O.Generator(CONFIGS[name]).state_dict().items()] == want
    assert [(k, tuple(v.shape)) for k, v in add_layers(nn.Module(), load_config(name)).state_dict().items()] == want
    assert [(k, tuple(v.shape)) for k, v in BigVGANVocoder(name).state_dict().items()] == want


def test_parameter_counts():
    counts = {n: sum(p.numel() for p in BigVGANVocoder(n).parameters()) for n in NAMES}
    print(f"\nbigvgan parameters: {counts}")
    assert counts == {"base_22khz_80band": 13953474, "22khz_80band": 112231250, "v2_22khz_80band_fmax8k_256x": 112231249}
    assert counts["base_22khz_80band"] == sum(p.numel() for p in O.Generator(CONFIGS["base_22khz_80band"]).parameters())


def test_flops_and_launches_per_config():
    got = {n: (BigVGANVocoder(n).flops_per_frame(), BigVGANVocoder(n).launches()) for n in NAMES}
    assert got == {"base_22khz_80band": (637501440, 160), "22khz_80band": (1833209856, 238),
                   "v2_22khz_80band_fmax8k_256x": (1833209856, 238)}
    # the activations' filters: 48 FLOP per channel and input row of each Activation1d
    base = BigVGANVocoder("base_22khz_80band")
    acts = 2 * 24 * (18 * (8 * 256 + 64 * 128 + 128 * 64 + 256 * 32) + 256 * 32)
    assert acts == 23396352                                           # tens of MFLOP per frame
    convs = (80 * 512 * 7 + 512 * 256 * 16 + 8 * 256 * 128 * 16 + 64 * 128 * 64 * 4 + 128 * 64 * 32 * 4      # conv_pre, ups
             + 6 * 21 * (8 * 256 ** 2 + 64 * 128 ** 2 + 128 * 64 ** 2 + 256 * 32 ** 2) + 256 * 32 * 7)          # resblocks, conv_post
    assert base.flops_per_frame() == acts + 2 * convs


def test_default_filters_are_the_kaiser_sinc_lowpass():
    f = kaiser_sinc_filter1d(0.25, 0.3, 12)
    assert f.shape == (1, 1, 12) and f.dtype == torch.float32
    ref = O.kaiser_sinc_filter1d(0.25, 0.3, 12, dtype=torch.float64)
    assert float((f.double() - ref).abs().max()) < 1e-7
    assert abs(float(ref.sum()) - 1) < 1e-12 and torch.allclose(ref, ref.flip(-1))
    assert bool((ref.abs() > 1e-4).all())                             # every tap counts: the reach of 5 is tight


def _act_by_index(x, fu, fd, alpha, inv):
    """Activation1d as csrc/bigvgan.cu computes it, element by element: u[m] = 2 sum_j x[clamp(j)] fu[m + 5 - 2 j], s[m] =
    u + inv sin^2(alpha u), out[t] = sum_k fd[k] s[clamp(2 t + k - 5)], clamps to the utterance.  x [C, n] float64."""
    C_, n = x.shape
    s = np.zeros((C_, 2 * n))
    for m in range(2 * n):
        p, odd = m >> 1, m & 1
        u = sum(x[:, min(max(p + 2 + odd - jj, 0), n - 1)] * fu[2 * jj + 1 - odd] for jj in range(6)) * 2
        s[:, m] = u + inv[:, 0] * np.sin(alpha[:, 0] * u) ** 2
    out = np.zeros((C_, n))
    for t in range(n):
        out[:, t] = sum(fd[k] * s[:, min(max(2 * t + k - 5, 0), 2 * n - 1)] for k in range(12))
    return out


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 6, 11, 40])
@pytest.mark.parametrize("beta", [False, True])
def test_activation_index_arithmetic_equals_the_oracle(n, beta):
    """The kernels' clamped index formula is the oracle's replicate-padded up / Snake / down chain, for utterances shorter
    than the replicate padding too, and output row t depends on input rows t - 5 .. t + 5 only."""
    torch.manual_seed(n)
    a = O.Activation1d(O.Snake(6, beta, True)).double()
    with torch.no_grad():
        a.act.alpha.uniform_(-1, 1)
        if beta:
            a.act.beta.uniform_(-1, 1)
        a.upsample.filter.mul_(1 + 0.01 * torch.rand(12, dtype=torch.float64))    # unsymmetric filters: no tap reversed
        a.downsample.lowpass.filter.mul_(1 + 0.01 * torch.rand(12, dtype=torch.float64))
    x = torch.randn(1, 6, n, dtype=torch.float64) * 3
    with torch.no_grad():
        want = a(x)[0].numpy()
    al = torch.exp(a.act.alpha.detach()).numpy()
    be = torch.exp(a.act.beta.detach()).numpy() if beta else al
    got = _act_by_index(x[0].numpy(), a.upsample.filter.flatten().numpy(), a.downsample.lowpass.filter.flatten().numpy(), al[:, None],
                        1 / (be[:, None] + 1e-9))
    assert want.shape == (6, n) and np.abs(got - want).max() < 1e-12
    if n >= 11:
        x2 = x.clone()
        x2[..., 5] = float("nan")
        with torch.no_grad():
            cone = torch.isnan(a(x2)[0, 0])
        assert cone.nonzero().flatten().tolist() == list(range(0, min(11, n)))


def _folded_forward(v: BigVGANVocoder, mel):
    """The generator in torch.nn.functional from BigVGANVocoder's folded weights, exp'd Snake parameters and filters
    (what fs2_bigvgan_load receives)."""
    cfg = v.config

    def conv(m, x, d=1):
        return F.conv1d(x, m.folded(), None if m.bias is None else m.bias.detach(), dilation=d, padding=d * (m.weight_v.shape[2] - 1) // 2)

    def act(a, x):
        C_ = x.shape[1]
        al = a.act.alpha.detach()
        be = al if a.act.beta is None else a.act.beta.detach()
        if cfg["snake_logscale"]:
            al, be = torch.exp(al), torch.exp(be)
        u = 2 * F.conv_transpose1d(F.pad(x, (5, 5), mode="replicate"), a.upsample.filter.expand(C_, -1, -1), stride=2, groups=C_)[..., 15:-15]
        s = u + 1 / (be[None, :, None] + 1e-9) * torch.sin(al[None, :, None] * u) ** 2
        return F.conv1d(F.pad(s, (5, 6), mode="replicate"), a.downsample.lowpass.filter.expand(C_, -1, -1), stride=2, groups=C_)

    x = conv(v.conv_pre, mel)
    nk = len(cfg["resblock_kernel_sizes"])
    for i, u in enumerate(cfg["upsample_rates"]):
        x = F.conv_transpose1d(x, v.ups[i][0].folded(), v.ups[i][0].bias.detach(), stride=u, padding=u // 2)
        xs = None
        for j in range(nk):
            rb, dil, y = v.resblocks[i * nk + j], cfg["resblock_dilation_sizes"][j], x
            if cfg["resblock"] == "1":
                for m, (c1, c2, d) in enumerate(zip(rb.convs1, rb.convs2, dil)):
                    y = conv(c2, act(rb.activations[2 * m + 1], conv(c1, act(rb.activations[2 * m], y), d))) + y
            else:
                for m, (c, d) in enumerate(zip(rb.convs, dil)):
                    y = conv(c, act(rb.activations[m], y), d) + y
            xs = y if xs is None else xs + y
        x = xs / nk
    y = conv(v.conv_post, act(v.activation_post, x))
    return torch.tanh(y) if cfg["use_tanh_at_final"] else torch.clamp(y, -1, 1)


@pytest.mark.parametrize("cfg", [dict(SMALL["base"]), dict(SMALL["base"], resblock="2", activation="snake", snake_logscale=False,
                                                                    use_tanh_at_final=False, use_bias_at_final=False)])
def test_folded_forward_equals_the_weight_norm_module(cfg):
    g = _perturbed(O.Generator(cfg), 1)
    v = BigVGANVocoder(cfg)
    v.load_state_dict(g.state_dict())
    mel = torch.randn(1, 80, 6) * 2 - 6
    with torch.no_grad():
        want = g(mel)
        got = _folded_forward(v, mel)
    assert got.shape == want.shape == (1, 1, 6 * 256)
    assert float((got - want).abs().max()) <= 1e-5                 # fp32 noise


def test_oracle_batched_is_per_utterance():
    """Utterances of 1 to 4 frames: every Activation1d replicate-pads wider than the utterance."""
    g = _perturbed(O.Generator(SMALL["base"]), 2)
    mels = torch.randn(5, 7, 80) * 2 - 6
    olens = [7, 1, 2, 3, 4]
    with torch.no_grad():
        audio = O.batched(g, mels, olens)
        for b, n in enumerate(olens):
            one = g(mels[b, :n].T[None])[0, 0]
            assert torch.equal(audio[b, : n * 256], one) and torch.all(audio[b, n * 256:] == 0)
            assert torch.isfinite(one).all()


def _with(name, **edits):
    cfg = json.loads(json.dumps(CONFIGS[name]))
    cfg.update(edits)
    return cfg


B_ = "base_22khz_80band"


@pytest.mark.parametrize("cfg,field", [
    (_with(B_, upsample_rates=[8, 8, 2, 4], upsample_kernel_sizes=[16, 16, 4, 8]), "upsample_rates"),
    (_with(B_, upsample_kernel_sizes=[16, 16, 4, 5]), "upsample_kernel_sizes"),
    (_with(B_, upsample_rates=[256 // 3, 3], upsample_kernel_sizes=[170, 6]), "upsample_rates"),
    (_with(B_, num_mels=100), "num_mels"),
    (_with(B_, num_mels=128), "num_mels"),
    (_with(B_, resblock="3"), "resblock"),
    (_with(B_, upsample_initial_channel=64), "upsample_initial_channel"),         # 64 / 16 = 4: not a multiple of 8
    (_with(B_, upsample_initial_channel=4096), "upsample_initial_channel"),
    (_with(B_, upsample_initial_channel=200), "upsample_initial_channel"),
    (_with(B_, resblock_kernel_sizes=[3, 6, 11]), "resblock_kernel_sizes"),
    (_with(B_, resblock_dilation_sizes=[[1], [1, 3, 5], [1, 3, 5]]), "resblock_dilation_sizes"),
    (_with(B_, activation="relu"), "activation"),
    (_with(B_, snake_logscale=1), "snake_logscale"),
    (_with(B_, use_tanh_at_final="no"), "use_tanh_at_final"),
    (_with(B_, upsample_initial_channel=128), None),                                # widths 128 ... 8
    (_with(B_, upsample_rates=[8, 4, 2, 2, 2], upsample_kernel_sizes=[16, 8, 4, 4, 4], upsample_initial_channel=768), None),   # ... 48, 24
    (_with(B_, resblock="2", activation="snake"), None),
])
def test_config_refusals_name_their_field(cfg, field):
    if field is None:
        check_config(load_config(cfg))
        return
    with pytest.raises(ValueError, match=field):
        BigVGANVocoder(cfg)


def test_config_forms_and_missing_fields(tmp_path):
    path = tmp_path / "config.json"
    path.write_text(json.dumps(dict(CONFIGS["v2_22khz_80band_fmax8k_256x"], sampling_rate=22050, fmax=8000, use_cqtd_instead_of_mrd=True)))
    v = BigVGANVocoder(str(path))
    assert v.config == BigVGANVocoder("v2_22khz_80band_fmax8k_256x").config
    assert v.config["use_tanh_at_final"] is False and v.config["use_bias_at_final"] is False
    assert BigVGANVocoder("22khz_80band").config["use_tanh_at_final"] is True
    assert "conv_post.bias" not in v.state_dict() and "conv_post.bias" in BigVGANVocoder("22khz_80band").state_dict()
    for field in ("activation", "snake_logscale", "resblock_dilation_sizes"):
        cfg = dict(CONFIGS[B_])
        del cfg[field]
        with pytest.raises(ValueError, match=field):
            BigVGANVocoder(cfg)
    with pytest.raises(ValueError, match="config"):
        BigVGANVocoder(42)
    with pytest.raises(ValueError, match="math_mode"):
        BigVGANVocoder(B_, math_mode="bf16")


def test_from_checkpoint_forms_and_config_discovery(tmp_path):
    cfg = SMALL["base"]
    g = _perturbed(O.Generator(cfg), 3)
    with torch.no_grad():
        g.activation_post.upsample.filter.mul_(1.5)                  # the checkpoint's filters are loaded, not recomputed
    sd = g.state_dict()
    d = tmp_path / "run"
    d.mkdir()
    path = d / "bigvgan_generator.pt"
    torch.save({"generator": sd}, path)
    with pytest.raises(ValueError, match="config"):
        BigVGANVocoder.from_checkpoint(str(path))                    # no config.json yet
    with pytest.raises(ValueError, match="config"):
        BigVGANVocoder.from_checkpoint({"generator": sd})
    (d / "config.json").write_text(json.dumps(cfg))
    for src, c in ((str(path), None), (path, None), ({"generator": sd}, cfg), (sd, cfg)):
        v = BigVGANVocoder.from_checkpoint(src, config=c)
        assert v.config == BigVGANVocoder(cfg).config
        assert all(torch.equal(v.state_dict()[k], sd[k]) for k in sd)
    g.remove_weight_norm()
    plain = g.state_dict()
    assert any(k.endswith(".weight") for k in plain) and not any(k.endswith("weight_g") for k in plain)
    v = BigVGANVocoder.from_checkpoint({"generator": plain}, config=cfg)
    for name, m in v.named_modules():
        if hasattr(m, "folded"):
            assert torch.equal(m.folded(), plain[f"{name}.weight"]), name
    with pytest.raises(ValueError, match="shape"):
        BigVGANVocoder.from_checkpoint(sd, config=dict(cfg, upsample_initial_channel=256))


V2 = "v2_22khz_80band_fmax8k_256x"


@pytest.mark.parametrize("name,edit,match", [
    (B_, lambda sd: sd.pop("resblocks.4.convs1.1.weight_v"), "missing key resblocks.4.convs1.1.weight_v"),
    (B_, lambda sd: sd.pop("resblocks.4.activations.3.act.beta"), "missing key resblocks.4.activations.3.act.beta"),
    (B_, lambda sd: sd.pop("activation_post.downsample.lowpass.filter"), "missing key activation_post.downsample.lowpass.filter"),
    (B_, lambda sd: sd.__setitem__("resblocks.0.activations.0.upsample.filter", torch.zeros(1, 1, 13)),
     r"resblocks.0.activations.0.upsample.filter has shape \(1, 1, 13\)"),
    (B_, lambda sd: sd.__setitem__("activation_post.act.alpha", torch.zeros(33)), "activation_post.act.alpha has shape"),
    (B_, lambda sd: sd.__setitem__("ups.0.0.weight_g", torch.ones(256, 1, 1)), r"ups.0.0.weight_g has shape \(256, 1, 1\)"),
    (B_, lambda sd: sd.__setitem__("resblocks.0.activations.6.act.alpha", torch.zeros(256)), "unexpected key resblocks.0.activations.6"),
    (V2, lambda sd: sd.__setitem__("conv_post.bias", torch.zeros(1)), "unexpected key conv_post.bias"),
])
def test_from_checkpoint_rejects_bad_keys_by_name(name, edit, match):
    sd = dict(O.Generator(CONFIGS[name]).state_dict())
    edit(sd)
    with pytest.raises(ValueError, match=match):
        BigVGANVocoder.from_checkpoint({"generator": sd}, config=name)


# ---- the window plan ------------------------------------------------------------------------------------------------

def test_plan_numbers_for_the_named_configs():
    for name in NAMES:
        cfg = CONFIGS[name]
        v = BigVGANVocoder(name)
        plan = v.window_plan()
        r = BP.reaches(cfg)
        U = len(cfg["upsample_rates"])
        assert plan["R"] == BP.stack_reach(cfg) == 90
        assert plan["reach"] == [r[f"ups{s}"] for s in range(U)]
        assert plan["halo"] == [BP.level_halo(cfg, s) for s in range(U + 1)]
        for level, wrong, spare in BP.exact_margins(cfg):
            assert wrong <= spare, (name, level, wrong, spare)
        assert v._window_rows(64, 32) == (64 * BP.level_rows(cfg, U, 32), f"B * (256 * n_frames + {2 * plan['halo'][U]})")
    assert BigVGANVocoder(B_).window_plan() == {"reach": [15, 21, 71, 50], "halo": [18, 120, 168, 142, 100], "R": 90}
    assert BigVGANVocoder("22khz_80band").window_plan() == {"reach": [35, 45, 86, 81, 71, 50], "halo": [38, 140, 180, 172, 162, 142, 100],
                                                           "R": 90}
    assert BP.workspace_bytes(CONFIGS[B_], 64, 32) == 390_610_176
    assert BP.whole_call_workspace_bytes(CONFIGS[B_], 4, 2000) - BP.whole_call_workspace_bytes(CONFIGS[B_], 4, 1000) == 163840 * 4000
    assert BP.whole_call_workspace_bytes(CONFIGS["22khz_80band"], 4, 2000) - BP.whole_call_workspace_bytes(CONFIGS["22khz_80band"], 4, 1000) \
        == 5 * 4 * 256 * 32 * 4000                                   # the 24-wide last stage is 32 wide in the buffers


def test_plan_is_exact_for_a_grid_of_accepted_configs():
    for resblock in ("1", "2"):
        for rates in ([8, 8, 2, 2], [4, 4, 2, 2, 2, 2], [8, 8, 4], [16, 16], [2] * 8):
            for kers, dils in (([3, 7, 11], [[1, 3, 5]] * 3), ([3, 5, 7], [[1, 2, 4], [2, 6, 8], [3, 12, 1]]), ([1], [[1, 1, 1]])):
                cfg = dict(CONFIGS[B_], resblock=resblock, upsample_rates=rates, upsample_kernel_sizes=[2 * u for u in rates],
                           upsample_initial_channel=8 << len(rates), resblock_kernel_sizes=kers, resblock_dilation_sizes=dils)
                check_config(load_config(cfg))
                plan = BigVGANVocoder(cfg).window_plan()
                assert plan["halo"] == [BP.level_halo(cfg, s) for s in range(len(rates) + 1)], cfg
                for level, wrong, spare in BP.exact_margins(cfg):
                    assert wrong <= spare, (cfg, level, wrong, spare)


@pytest.mark.parametrize("topology,name", [("base", B_), ("large", "22khz_80band")])
def test_plan_reach_matches_the_nan_cone(topology, name):
    """A NaN at mel frame c0 - h_0 reaches the audio of the window [c0, c1), one at c0 - h_0 - 1 does not, and the same on
    the right (c1 - 1 + h_0, c1 + h_0): the float64 oracle at reduced widths (the large topology with a 24-wide stage)."""
    h0 = BigVGANVocoder(name).window_plan()["halo"][0]
    cfg = SMALL[topology]
    assert topology == "base" or 24 in BP.widths(cfg)
    g = _perturbed(O.Generator(cfg), 4).double()
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


# ---- the C entry points ---------------------------------------------------------------------------------------------

def test_library_exports_bigvgan_entry_points():
    lib = _lib.load()
    header = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    for name in ("fs2_bigvgan_create", "fs2_bigvgan_load", "fs2_bigvgan_workspace_bytes", "fs2_bigvgan", "fs2_bigvgan_window_workspace_bytes",
                 "fs2_bigvgan_window", "fs2_op_bigvgan_act", "fs2_op_bigvgan_resblock"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES, name
        assert f"int {name}(" in header, name
    assert hasattr(lib, "fs2_bigvgan_destroy") and "void fs2_bigvgan_destroy(" in header
    for k in ("BAD_LENGTH", "RANGE", "BAD_START", "SNAKE", "SNAKEBETA"):
        assert int(re.search(rf"#define FS2_BIGVGAN_{k} (\d+)", header).group(1)) == getattr(_lib, f"FS2_BIGVGAN_{k}")


def test_create_validates_the_config_in_c():
    """fs2_bigvgan_create refuses what check_config refuses, before it touches the device, naming the field."""
    lib = _lib.load()
    base = BigVGANVocoder(B_)

    def create(**edits):
        c = base._c_config()
        for k, v in edits.items():
            if k == "rate":
                c.gen.upsample_rates[0] = v
            elif k == "kernel":
                c.gen.upsample_kernel_sizes[0] = v
            elif k == "rk":
                c.gen.resblock_kernel_sizes[0] = v
            elif k == "dil":
                c.gen.resblock_dilation_sizes[0][0] = v
            elif k == "activation":
                c.activation = v
            else:
                setattr(c.gen, k, v)
        h = C.c_void_p()
        return lib.fs2_bigvgan_create(C.byref(h), _lib.MATH_3XTF32, C.byref(c))

    for edits, what in ((dict(resblock=3), b"resblock"), (dict(rate=4, kernel=8), b"product"), (dict(kernel=15), b"upsample_kernel_sizes"),
                        (dict(rate=7, kernel=14), b"upsample_rates"), (dict(upsample_initial_channel=64), b"upsample_initial_channel"),
                        (dict(upsample_initial_channel=4096), b"upsample_initial_channel"),
                        (dict(upsample_initial_channel=200), b"upsample_initial_channel"), (dict(num_upsamples=0), b"num_upsamples"),
                        (dict(rk=4), b"resblock_kernel_sizes"), (dict(dil=0), b"resblock_dilation_sizes"),
                        (dict(num_dilations=2), b"num_dilations"), (dict(num_kernels=9), b"num_kernels"), (dict(activation=2), b"activation")):
        assert create(**edits) == -1, edits
        assert what in lib.fs2_last_error(), (edits, lib.fs2_last_error())


def test_single_layer_entries_reject_bad_arguments_on_the_host():
    lib = _lib.load()
    p = 256
    wp = (C.c_void_p * 24)(*([p] * 24))

    def block(mode=_lib.MATH_3XTF32, type_=2, C_=64, k=3, dils=(1, 3), x=p, out=p, B=2, Lp=40):
        d = (C.c_int * len(dils))(*dils)
        return lib.fs2_op_bigvgan_resblock(mode, type_, C_, k, len(dils), d, x, p, B, Lp, wp, wp, wp, 1, 1, out, p, None)

    def act(mode=_lib.MATH_3XTF32, C_=24, x=p, B=2, Lp=40, snakebeta=1, tensors=wp):
        return lib.fs2_op_bigvgan_act(mode, C_, x, p, B, Lp, tensors, snakebeta, 1, p, p, None)

    for mode in (-1, 4):
        assert block(mode=mode) == -1 and b"math_mode" in lib.fs2_last_error()
        assert act(mode=mode) == -1 and b"math_mode" in lib.fs2_last_error()
    assert block(type_=3) == -1 and b"type" in lib.fs2_last_error()
    for C_ in (0, 16, 48, 80):
        assert block(C_=C_) == -1 and b"C must be" in lib.fs2_last_error()
    assert block(type_=1, dils=(1, 3)) == -1 and b"nd must be" in lib.fs2_last_error()
    assert block(x=p + 8) == -1 and b"aligned" in lib.fs2_last_error()
    assert block(mode=_lib.MATH_FP32, B=65535, Lp=129) == -1 and b"too many rows" in lib.fs2_last_error()
    for C_ in (0, 12, 2056):
        assert act(C_=C_) == -1 and b"C must be" in lib.fs2_last_error()
    assert act(x=None) == -1 and b"null" in lib.fs2_last_error()
    nobeta = (C.c_void_p * 4)(p, None, p, p)
    assert act(tensors=nobeta) == -1 and b"null" in lib.fs2_last_error()
    assert act(Lp=0) == -1 and b"shape" in lib.fs2_last_error()


def test_bigvgan_kernels_do_not_spill():
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "bigvgan.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = open(reports[0]).read()
    # the Activation1d kernels only: BigVGAN's chain runs on hifigan.cu's, its padding pack is vocoder_weights.cu's
    expected = {"bigvgan_act_kernel": 3, "bigvgan_post_kernel": 1, "act_param_kernel": 1}
    for kernel, n in expected.items():
        props = re.findall(r"Function properties for \S*%s\S*\n(.*)" % kernel, text)
        assert len(props) == n, (kernel, len(props))
        for line in props:
            assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in line, (kernel, line)
    assert len(re.findall(r"Function properties for ", text)) == sum(expected.values())
