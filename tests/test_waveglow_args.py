"""WaveGlow vocoder without a GPU: the CPU oracle's keys against tests/golden/waveglow_state_dict_keys.json, its
internal consistency (infer inverts forward, the batched restatement is per-utterance infer), checkpoint loading in both
key sets with the DeepLearningExamples wrapper and prefix, the torch.hub hook of the drop-in launcher, argument
validation, the C entry points and the ptxas report of the new kernels."""
import glob
import json
import os
import re
import subprocess
import sys

import pytest
import torch

from conftest import GOLDEN, REPO
from fastspeech2_b200 import _lib
from fastspeech2_b200 import dropin_run
from fastspeech2_b200.waveglow import WaveGlowVocoder, flow_channels
from oracle import waveglow_oracle as O


def _golden():
    return [(k, tuple(s)) for k, s in json.load(open(os.path.join(GOLDEN, "waveglow_state_dict_keys.json")))]


def _oracle(C, seed=0):
    """Weights far from the published init: g moved away from |v|, and `end` non-zero (a zero `end` makes every coupling
    the identity)."""
    torch.manual_seed(seed)
    g = O.WaveGlow(C)
    with torch.no_grad():
        for name, p in g.named_parameters():
            if name.endswith("weight_g"):
                p.mul_(torch.rand(p.shape) + 0.5)
        for wn in g.WN:
            wn.end.weight.normal_(0, 1.0 / C ** 0.5)
            wn.end.bias.normal_(0, 0.1)
    return g.eval()


def test_oracle_keys_match_the_golden_list():
    g = O.WaveGlow(512)
    sd = g.state_dict()
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == _golden()
    assert len(sd) == 938 == 12 * 77 + 12 + 2
    assert sum(p.numel() for p in g.parameters()) == 268294760
    assert [O.flow_channels(k) for k in range(12)] == [8, 8, 8, 8, 6, 6, 6, 6, 4, 4, 4, 4]
    assert [tuple(sd[f"convinv.{k}.conv.weight"].shape) for k in range(12)] == [(c, c, 1) for c in map(O.flow_channels, range(12))]


def test_vocoder_parameters_carry_the_same_keys():
    v = WaveGlowVocoder(512)
    assert [(k, tuple(t.shape)) for k, t in v.state_dict().items()] == _golden()


def test_oracle_infer_inverts_forward_in_float64():
    g = _oracle(32, 1).double()
    T = 6
    mel = torch.randn(1, 80, T, dtype=torch.float64) * 2 - 6
    audio = torch.randn(1, T * 256, dtype=torch.float64) * 0.3
    with torch.no_grad():
        z = g.forward(mel, audio)
        back = g.infer(mel, 1.0, z)
        s = g.WN[11](z[:, 4:6], g._cond(mel, T * 32))[:, 2:]
    assert z.shape == (1, 8, T * 32)
    assert float(s.abs().mean()) > 0.1                  # the couplings are far from the identity
    assert float((back - audio).abs().max()) <= 1e-9
    # sigma scales the draw: infer(z / sigma, sigma) is infer(z)
    with torch.no_grad():
        assert float((g.infer(mel, 0.5, z / 0.5) - audio).abs().max()) <= 1e-9


def test_oracle_batched_is_per_utterance_infer():
    g = _oracle(32, 2).double()
    olens = [5, 2, 3]
    mels = torch.randn(3, 5, 80, dtype=torch.float64) * 2 - 6
    z = torch.randn(3, 8, 5 * 32, dtype=torch.float64)
    with torch.no_grad():
        out = O.batched(g, mels, olens, z, sigma=0.8)
        for b, n in enumerate(olens):
            one = g.infer(mels[b, :n].T[None], 0.8, z[b: b + 1, :, : n * 32])
            assert torch.equal(out[b, : n * 256], one[0])
            assert torch.all(out[b, n * 256:] == 0)
    # torch.randn noise, as DeepLearningExamples draws it: reproducible under torch.manual_seed
    torch.manual_seed(3)
    a = g.infer(mels[:1].transpose(1, 2), 1.0)
    torch.manual_seed(3)
    assert torch.equal(a, g.infer(mels[:1].transpose(1, 2), 1.0)) and a.shape == (1, 5 * 256)


def _clone(g):
    c = O.WaveGlow(g.WN[0].n_channels)                 # deepcopy does not take weight-normed modules
    c.load_state_dict(g.state_dict())
    return c.eval()


def _plain(g):
    return O.WaveGlow.remove_weightnorm(_clone(g)).state_dict()


@pytest.mark.parametrize("C", [256, 512])
def test_from_checkpoint_accepts_both_key_sets_the_wrapper_and_the_prefix(tmp_path, C):
    g = _oracle(C, 3)
    sd = g.state_dict()
    path = tmp_path / "waveglow.pt"
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}, "epoch": 1, "config": {}}, path)
    for src in (sd, {"state_dict": sd}, str(path)):
        v = WaveGlowVocoder.from_checkpoint(src)
        assert v.n_channels == C
        assert all(torch.equal(v.state_dict()[k], sd[k]) for k in sd)
    plain = _plain(g)
    assert any(k.endswith("start.weight") for k in plain) and not any(k.endswith("weight_g") for k in plain)
    v = WaveGlowVocoder.from_checkpoint({"state_dict": {"module." + k: t for k, t in plain.items()}})
    for name, m in v.named_modules():
        if hasattr(m, "folded"):
            w = plain[f"{name}.weight"]
            assert float((m.folded() - w).abs().max()) <= 1e-6 * float(w.abs().max()), name


@pytest.mark.parametrize("edit,match", [
    (lambda sd: sd.pop("WN.3.in_layers.5.weight_v"), "missing key WN.3.in_layers.5.weight_v"),
    (lambda sd: sd.pop("convinv.7.conv.weight"), "missing key convinv.7.conv.weight"),
    (lambda sd: sd.__setitem__("WN.0.cond_layer.weight", torch.zeros(3)), "unexpected key WN.0.cond_layer.weight"),
    (lambda sd: sd.__setitem__("WN.2.end.weight", torch.zeros(4, 256, 1)), r"WN.2.end.weight has shape \(4, 256, 1\)"),
    (lambda sd: sd.__setitem__("WN.4.in_layers.0.weight_v", torch.zeros(1024, 512, 3)), "WN.4.in_layers.0.weight_v has shape"),
    (lambda sd: sd.__setitem__("WN.9.start.bias", torch.zeros(512)), "WN.9.start.bias has shape"),
    (lambda sd: sd.__setitem__("upsample.weight", torch.zeros(80, 80, 512)), "upsample.weight has shape"),
    (lambda sd: sd.pop("WN.0.start.bias"), "missing key WN.0.start.bias"),
])
def test_from_checkpoint_rejects_bad_keys_by_name(edit, match):
    sd = dict(O.WaveGlow(256).state_dict())
    edit(sd)
    with pytest.raises(ValueError, match=match):
        WaveGlowVocoder.from_checkpoint({"state_dict": sd})


def test_inconsistent_or_unsupported_channels_raise():
    sd = dict(O.WaveGlow(256).state_dict())
    sd["WN.0.start.bias"] = torch.zeros(100)
    with pytest.raises(ValueError, match="n_channels"):
        WaveGlowVocoder.from_checkpoint(sd)
    with pytest.raises(ValueError, match="n_channels"):
        WaveGlowVocoder(n_channels=96)


@pytest.fixture
def fake_hub(monkeypatch):
    calls = []
    monkeypatch.setattr(torch.hub, "load", lambda repo, model, *a, **k: calls.append((repo, model)) or "original")
    return calls


def test_dropin_hook_serves_only_nvidia_waveglow(tmp_path, fake_hub):
    path = tmp_path / "w.pt"
    torch.save({"state_dict": O.WaveGlow(256).state_dict()}, path)
    dropin_run.install_waveglow_hub(str(path))
    v = torch.hub.load("nvidia/DeepLearningExamples:torchhub", "nvidia_waveglow", model_math="fp32")
    assert isinstance(v, WaveGlowVocoder) and v.math_mode == "3xf16" and v.n_channels == 256
    assert torch.hub.load("NVIDIA/DeepLearningExamples", "nvidia_waveglow", model_math="fp16").math_mode == "f16"
    assert v.remove_weightnorm(v) is v
    with pytest.raises(ValueError, match="pretrained"):
        torch.hub.load("nvidia/DeepLearningExamples:torchhub", "nvidia_waveglow", pretrained=False)
    assert torch.hub.load("nvidia/DeepLearningExamples:torchhub", "nvidia_tacotron2") == "original"
    assert torch.hub.load("seungwonpark/melgan", "melgan") == "original"
    assert fake_hub == [("nvidia/DeepLearningExamples:torchhub", "nvidia_tacotron2"), ("seungwonpark/melgan", "melgan")]


@pytest.mark.parametrize("order", ["melgan first", "waveglow first"])
def test_melgan_and_waveglow_hooks_compose_in_either_order(tmp_path, fake_hub, order):
    from fastspeech2_b200.melgan import MelGANVocoder
    from oracle import melgan_oracle
    wpath, mpath = tmp_path / "w.pt", tmp_path / "m.pt"
    torch.save({"state_dict": O.WaveGlow(256).state_dict()}, wpath)
    torch.save({"model_g": melgan_oracle.Generator().state_dict()}, mpath)
    installs = [lambda: dropin_run.install_melgan_hub(str(mpath)), lambda: dropin_run.install_waveglow_hub(str(wpath))]
    for install in installs if order == "melgan first" else installs[::-1]:
        install()
    assert isinstance(torch.hub.load("seungwonpark/melgan", "melgan"), MelGANVocoder)
    assert isinstance(torch.hub.load("nvidia/DeepLearningExamples:torchhub", "nvidia_waveglow"), WaveGlowVocoder)
    assert torch.hub.load("nvidia/DeepLearningExamples:torchhub", "nvidia_tacotron2") == "original"
    assert fake_hub == [("nvidia/DeepLearningExamples:torchhub", "nvidia_tacotron2")]


def test_dilated_tap_gemm_entry_bounds_the_dilation():
    """fs2_op_tap_gemm_dil refuses these before it touches memory (the pointers are never dereferenced): the tap rows
    t + (j - pad) * dil must stay int32 row coordinates."""
    lib = _lib.load()
    p = 256

    def call(dil, taps=3, L=100):
        return lib.fs2_op_tap_gemm_dil(_lib.MATH_FP32, p, 2, L, 64, p, None, 64, taps, 0, None, None, p, None, 0, 0, None, 0,
                                       dil, None)

    assert call(0) == -1 and call(-4) == -1
    assert call(2 ** 30) == -1 and call(2 ** 30 - 100, taps=3, L=100) == -1 and call(2 ** 29, taps=5) == -1
    assert b"dil" in lib.fs2_last_error()


def test_dropin_launcher_installs_the_hook_from_the_environment(tmp_path):
    path = tmp_path / "w.pt"
    torch.save({"state_dict": {"module." + k: v for k, v in O.WaveGlow(256).state_dict().items()}}, path)
    script = tmp_path / "uses_hub.py"
    script.write_text("import torch\n"
                      "w = torch.hub.load('nvidia/DeepLearningExamples:torchhub', 'nvidia_waveglow', model_math='fp16')\n"
                      "w = w.remove_weightnorm(w)\n"
                      "print(type(w).__name__, len(w.state_dict()), w.math_mode, w.n_channels)\n")
    env = dict(os.environ, FS2_WAVEGLOW_CHECKPOINT=str(path), PYTHONPATH=REPO)
    r = subprocess.run([sys.executable, "-m", "fastspeech2_b200.dropin_run", str(script)], cwd=str(tmp_path), env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert r.stdout.split() == ["WaveGlowVocoder", "938", "f16", "256"]


@pytest.fixture(scope="module")
def voc():
    return WaveGlowVocoder(256)


@pytest.mark.parametrize("shape,olens,match", [
    ((2, 10), [10, 9], "mels"), ((2, 10, 40), [10, 9], "mels"), ((0, 10, 80), [], "mels"), ((2, 10, 80), [10], "olens"),
    ((2, 10, 80), [10.0, 9.0], "integer"), ((2, 10, 80), [10, 9], "CUDA")])
def test_bad_inputs_raise(voc, shape, olens, match):
    with pytest.raises(ValueError, match=match):
        voc(torch.zeros(shape), torch.tensor(olens))


def test_integer_mels_raise(voc):
    with pytest.raises(ValueError, match="floating"):
        voc(torch.zeros(2, 10, 80, dtype=torch.int64), torch.tensor([10, 9]))


@pytest.mark.parametrize("kw,match", [
    (dict(sigma=float("nan")), "sigma"), (dict(sigma=float("inf")), "sigma"), (dict(sigma=-0.1), "sigma"), (dict(sigma="1"), "sigma"),
    (dict(z=torch.zeros(2, 8, 319)), "z must be"), (dict(z=torch.zeros(2, 6, 320)), "z must be"),
    (dict(z=torch.zeros(2, 8, 320, dtype=torch.int32)), "z must be"), (dict(z=torch.zeros(2, 8, 320), seed=1), "either z or seed"),
    (dict(seed=torch.tensor([1, 2, 3])), "seed"), (dict(seed=torch.tensor([1.0, 2.0])), "seed"), (dict(seed=1.5), "seed"),
    (dict(seed=2 ** 63), "int64"), (dict(seed=True), "seed"),
    (dict(z=torch.zeros(2, 8, 320)), "CUDA"), (dict(seed=3), "CUDA")])
def test_bad_noise_arguments_raise(voc, kw, match):
    with pytest.raises(ValueError, match=match):
        voc(torch.zeros(2, 10, 80), torch.tensor([10, 9]), **kw)


def test_noise_arguments_are_validated():
    with pytest.raises(ValueError, match="olens"):
        WaveGlowVocoder.noise(torch.tensor([3, 2]), 4, 0)           # CPU
    with pytest.raises(ValueError, match="seed"):
        WaveGlowVocoder._seeds(torch.tensor([[1, 2]]), 2, "cpu")
    assert torch.equal(WaveGlowVocoder._seeds(2 ** 63 - 1, 2, "cpu"), torch.tensor([2 ** 63 - 1, -2 ** 63]))   # wraps
    torch.manual_seed(5)
    a = WaveGlowVocoder._seeds(None, 3, "cpu")
    torch.manual_seed(5)
    assert torch.equal(a, WaveGlowVocoder._seeds(None, 3, "cpu")) and torch.equal(a - a[0], torch.arange(3))


def test_size_limits_raise_value_error():
    v = WaveGlowVocoder(256, math_mode="fp32")
    with pytest.raises(ValueError, match="fp32"):
        v._check_size(1, 65535 * 128 // 32 + 1)
    v._check_size(1, 65535 * 128 // 32)
    t = WaveGlowVocoder(256, math_mode="tf32")
    t._check_size(1, 65535 * 128 // 32 + 1)
    with pytest.raises(ValueError, match="2\\^31"):
        t._check_size(64, 2 ** 31 // 32 // 64)


def test_bad_math_mode_and_infer_shape_raise(voc):
    with pytest.raises(ValueError, match="math_mode"):
        WaveGlowVocoder(256, math_mode="bf16")
    with pytest.raises(ValueError, match="spect"):
        voc.infer(torch.zeros(1, 5, 80))


def test_load_tensors_are_in_the_c_order():
    """fs2_waveglow_load's 638 tensors: upsample, then per flow start, 8 in, 8 cond, 8 res_skip, end, W^-1 (float64)."""
    g = _oracle(64, 4)
    v = WaveGlowVocoder(64)
    v.load_state_dict(g.state_dict())
    ts = v._tensors()
    assert len(ts) == 2 + 12 * 53
    assert tuple(ts[0].shape) == (80, 80, 1024) and tuple(ts[2].shape) == (64, 4, 1)
    k = 11
    base = 2 + k * 53
    assert tuple(ts[base].shape) == (64, 2, 1) and tuple(ts[base + 2].shape) == (128, 64, 3)
    assert tuple(ts[base + 18].shape) == (128, 640, 1) and tuple(ts[base + 34 + 14].shape) == (64, 64, 1)
    W = g.convinv[k].conv.weight.detach().double()[:, :, 0]
    assert torch.equal(ts[base + 52], torch.linalg.inv(W).float())
    assert float((ts[base + 52].double() @ W - torch.eye(4, dtype=torch.float64)).abs().max()) < 1e-6
    w = g.WN[k].in_layers[3]
    assert torch.equal(ts[base + 2 + 6], torch._weight_norm(w.weight_v.detach(), w.weight_g.detach(), 0))


def test_library_exports_waveglow_entry_points():
    lib = _lib.load()
    header = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    for name in ("fs2_waveglow_create", "fs2_waveglow_load", "fs2_waveglow_workspace_bytes", "fs2_waveglow", "fs2_waveglow_noise",
                 "fs2_op_tap_gemm_dil", "fs2_op_waveglow_upsample", "fs2_op_waveglow_flow"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES, name
        assert f"int {name}(" in header, name
    assert hasattr(lib, "fs2_waveglow_destroy") and "void fs2_waveglow_destroy(" in header


def test_waveglow_kernels_beside_the_shared_prep_do_not_spill():
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "waveglow.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = open(reports[0]).read()
    # instantiations: noise, pack_taps, pack_up, add (1 each), the up operand, start and gate (3 operand kinds), the
    # cond planes (2 plane kinds), the flow kernel (n_half 2, 3, 4); the prep kernel is the window layer's
    expected = {"wg_noise_kernel": 1, "wg_pack_taps_kernel": 1, "wg_pack_up_kernel": 1, "wg_add_kernel": 1,
                "wg_up_operand_kernel": 3, "wg_start_kernel": 3, "wg_gate_kernel": 3, "wg_planes_kernel": 2, "wg_flow_kernel": 3}
    for kernel, n in expected.items():
        props = re.findall(r"Function properties for \S*%s\S*\n(.*)" % kernel, text)
        assert len(props) == n, (kernel, len(props))
        for line in props:
            assert "0 bytes spill stores, 0 bytes spill loads" in line, (kernel, line)


# ---- the per-stage entries (tests/test_gpu_waveglow_kernels.py) ----------------------------------------------------
def _flow(k=0, cond=256, skip=None, state_in=256, state_out=256, lens=256, B=2, Ls=40, wn=None, status=256, h=None):
    return _lib.load().fs2_op_waveglow_flow(h, k, cond, skip, state_in, state_out, lens, B, Ls, wn, status, None)


def _upsample(mels=256, olens=256, B=2, Lmax=5, cond=256, planes=None, status=256, h=None):
    return _lib.load().fs2_op_waveglow_upsample(h, mels, olens, B, Lmax, cond, planes, status, None)


@pytest.mark.parametrize("kw,match", [
    (dict(state_in=None), "null argument"), (dict(state_out=None), "null argument"), (dict(lens=None), "null argument"),
    (dict(status=None), "null argument"), (dict(cond=None), "null argument"),
    (dict(skip=256, wn=512), "wn_out needs the WN"),
    (dict(k=-1), "flow k"), (dict(k=12), "flow k"),
    (dict(B=0), "B >= 1 and Ls >= 1"), (dict(Ls=0), "B >= 1 and Ls >= 1"), (dict(Ls=-3), "B >= 1 and Ls >= 1"),
    (dict(cond=260), "16-byte aligned"), (dict(skip=264, cond=None), "16-byte aligned"), (dict(state_in=257), "16-byte aligned"),
    (dict(state_out=260), "16-byte aligned"), (dict(wn=268), "16-byte aligned"),
    ({}, "null or unloaded handle"), (dict(skip=256, cond=None), "null or unloaded handle")])
def test_flow_entry_refuses_on_the_host(kw, match):
    """fs2_op_waveglow_flow refuses these before it touches memory (the pointers are never dereferenced); the checks that
    need no handle run first, so each refusal names its own cause.  An unloaded handle and the row limits are checked on
    the GPU (test_gpu_waveglow_kernels.test_refusals_that_need_a_handle)."""
    assert _flow(**kw) == -1
    assert match.encode() in _lib.load().fs2_last_error()


@pytest.mark.parametrize("kw,match", [
    (dict(mels=None), "null argument"), (dict(olens=None), "null argument"), (dict(cond=None), "null argument"),
    (dict(status=None), "null argument"), (dict(B=0), "B >= 1 and Lmax >= 1"), (dict(Lmax=0), "B >= 1 and Lmax >= 1"),
    (dict(mels=264), "16-byte aligned"), (dict(cond=260), "16-byte aligned"), (dict(planes=258), "16-byte aligned"),
    ({}, "null or unloaded handle")])
def test_upsample_entry_refuses_on_the_host(kw, match):
    assert _upsample(**kw) == -1
    assert match.encode() in _lib.load().fs2_last_error()


def test_gpu_case_table_covers_the_tile_widths_flow_widths_and_lengths():
    """What the per-stage GPU cases reach, restated from the tap GEMM's schedule (tests/test_gpu_tap_gemm.py): res / skip
    GEMMs (N = C) on 64-, 80- and 128-wide tiles, every flow width, an utterance shorter than each dilation 2^i and not
    shorter than 2^(i-1), the lengths around one and two row tiles, Ls off the 128-row grid, and a case whose in-layer
    GEMM has more than 2 x 132 row tiles."""
    from test_gpu_tap_gemm import H100_SMS, tile_coords, tile_width, tiling
    import test_gpu_waveglow_kernels as K
    assert {tile_width(C) for C in K.WN_CS} == {64, 80, 128}        # the whole-flow cases run the GEMMs
    assert [tile_width(C) for C in K.WN_CS] == [64, 64, 128, 80, 128, 128]
    assert set(K.WN_CS) <= set(K.TAIL_CS) and {448, 960} <= set(K.TAIL_CS)   # wg_flow_kernel alone at more widths
    assert 1024 in K.WN_CS and 1024 in K.TAIL_CS                    # wg_flow_kernel's largest shared memory
    assert all(C % 64 == 0 and 64 <= C <= 1024 for C in K.WN_CS + K.TAIL_CS)
    assert {flow_channels(k) for k in K.FLOWS} == {4, 6, 8} and O.flow_channels(11) == 4
    assert {0, 1, 31, 127, 128, 129, 255, 257} <= set(K.LENS) and max(K.LENS) <= K.LS
    for i in range(1, 8):                                             # dilations 2 .. 128
        assert any(2 ** (i - 1) <= n < 2 ** i for n in K.LENS), i
    assert K.LS % 128 != 0
    B, Ls = K.BIG
    assert len(K.BIG_LENS) == B and max(K.BIG_LENS) <= Ls
    t = tiling(B, Ls, 2 * 256, 3, True)                               # the in-layer GEMM of the big case (C = 256)
    assert t.m_tiles == 3 * 94 and not t.packed
    live = [mt for mt in range(t.m_tiles) if not tile_coords(t, mt * t.n_tiles, K.BIG_LENS)[3]]
    assert len(live) == 94 + 93 + 86 > 2 * H100_SMS                   # live row tiles, not only walked ones
    assert tiling(len(K.LENS), K.LS, 256, 3, True).packed            # the 44-row tails share packed tiles
    assert min(K.UP_OLENS) == 0 and {1, 2, 3} <= set(K.UP_OLENS)
