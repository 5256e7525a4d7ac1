"""The ECAPA-TDNN encoder without a GPU (DESIGN.md section 28): the oracle's keys and shapes against
tests/golden/ecapa_state_dict_keys.json, checkpoint validation, the architecture read off the shapes, the front end
against a numpy float64 restatement, argument and size checks, the C entries' refusals and the ptxas report."""
import ctypes as C
import glob
import json
import os

import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib
from fastspeech2_b200.ecapa import ECAPAEncoder, architecture, expected_shapes, ordered_tensors
from oracle import ecapa_oracle as EO

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = json.load(open(os.path.join(REPO, "tests", "golden", "ecapa_state_dict_keys.json")))


def small(**kw):
    return EO.ECAPA_TDNN(**{"channels": (256, 256, 256, 256, 768), **kw})


@pytest.mark.parametrize("C", [1024, 512])
def test_oracle_keys_and_shapes_equal_the_json(C):
    kw = {} if C == 1024 else {"channels": (C, C, C, C, 3 * C)}
    sd = EO.ECAPA_TDNN(**kw).state_dict()
    assert {k: list(v.shape) for k, v in sd.items()} == KEYS[str(C)]
    assert list(sd) == list(KEYS[str(C)])
    want = {k: tuple(v) for k, v in KEYS[str(C)].items() if not k.endswith("num_batches_tracked")}
    assert expected_shapes(architecture(want)) == want
    for k in ("blocks.0.conv.conv.weight", "blocks.1.res2net_block.blocks.0.norm.norm.running_var", "blocks.2.se_block.conv1.conv.bias",
              "mfa.conv.conv.weight", "asp.tdnn.conv.conv.weight", "asp.conv.conv.bias", "asp_bn.norm.running_mean", "fc.conv.weight"):
        assert k in sd, k


def test_architecture_is_read_off_the_shapes():
    m = EO.ECAPA_TDNN(input_size=64, channels=(384, 384, 384, 1152), kernel_sizes=(3, 5, 5, 1), dilations=(1, 2, 3, 1),
                      attention_channels=64, res2net_scale=4, se_channels=32, lin_neurons=256, global_context=False)
    a = architecture({k: tuple(v.shape) for k, v in m.state_dict().items()}, dilations=(1, 2, 3, 1))
    assert a == {"n_mels": 64, "channels": 384, "n_blocks": 2, "scale": 4, "kernel_sizes": [3, 5, 5, 1], "dilations": [1, 2, 3, 1],
                 "se_channels": 32, "attention_channels": 64, "mfa_channels": 1152, "lin_neurons": 256, "global_context": False}
    enc = ECAPAEncoder(m.state_dict(), "fp32", dilations=(1, 2, 3, 1))
    assert enc.dim == 256 and enc.min_frames == 7 and enc.min_samples == 960      # block 2: k = 5 at d = 3 pads 6


def test_default_model_needs_640_samples():
    enc = ECAPAEncoder(small().state_dict())
    assert enc.min_samples == 640 and enc.min_frames == 5


def test_checkpoint_key_errors_name_the_key(tmp_path):
    sd = small().state_dict()
    bad = dict(sd); del bad["blocks.2.tdnn2.norm.norm.running_var"]
    with pytest.raises(ValueError, match="missing key blocks.2.tdnn2.norm.norm.running_var"):
        ECAPAEncoder(bad)
    bad = dict(sd); bad["blocks.1.extra"] = torch.zeros(1)
    with pytest.raises(ValueError, match="unexpected key blocks.1.extra"):
        ECAPAEncoder(bad)
    bad = dict(sd); bad["asp.conv.conv.bias"] = torch.zeros(5)
    with pytest.raises(ValueError, match="key asp.conv.conv.bias has shape"):
        ECAPAEncoder(bad)
    bad = {k: v for k, v in sd.items() if not k.endswith("num_batches_tracked")}
    ECAPAEncoder(bad)                                              # num_batches_tracked is optional
    torch.save(sd, tmp_path / "embedding_model.ckpt")
    assert ECAPAEncoder.from_checkpoint(str(tmp_path / "embedding_model.ckpt")).arch["channels"] == 256
    with pytest.raises(ValueError, match="math_mode"):
        ECAPAEncoder(sd, "bf16")


def test_channels_must_be_a_multiple_of_16_scale():
    m = EO.ECAPA_TDNN(channels=(200, 200, 200, 200, 600), res2net_scale=8)
    with pytest.raises(ValueError, match="multiple of 16"):
        ECAPAEncoder(m.state_dict())


def test_front_end_equals_numpy_float64():
    g = np.random.default_rng(0)
    x = g.standard_normal(5000) * 0.1
    x[1000:2600] = 0.0
    N, hop = 400, 160
    w = 0.54 - 0.46 * np.cos(2 * np.pi * np.arange(N) / N)
    xp = np.pad(x, (N // 2, N // 2))
    T = 1 + len(x) // hop
    frames = np.stack([xp[t * hop: t * hop + N] * w for t in range(T)])
    p = np.abs(np.fft.rfft(frames, axis=1)) ** 2
    mel = lambda f: 2595 * np.log10(1 + f / 700)                  # noqa: E731
    hz = 700 * (10 ** (np.linspace(0, mel(8000), 82) / 2595) - 1)
    fc, band = hz[1:-1], (hz[1:] - hz[:-1])[:-1]
    f = np.linspace(0, 8000, 201)
    sl = (f[:, None] - fc) / band
    fb = np.maximum(0, np.minimum(1 + sl, 1 - sl))
    db = 10 * np.log10(np.maximum(p @ fb, 1e-10))
    db = np.maximum(db, db.max() - 80)
    want = db - db.mean(0)
    got = EO.features(torch.from_numpy(x)).numpy()
    assert got.shape == (T, 80)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-9)
    assert (EO.fbank_db(torch.from_numpy(x)).numpy() >= db.max() - 80 - 1e-9).all()


def test_global_context_fold_is_exact_in_float64():
    m = small().double()
    x = torch.randn(768, 30, dtype=torch.float64)
    with torch.no_grad():
        assert torch.allclose(m.asp(x), m.asp(x, fold=True), rtol=1e-12, atol=1e-12)


def test_ordered_tensors_match_the_c_entry_count():
    for kw in ({}, {"res2net_scale": 4}):
        m = small(**kw)
        enc = ECAPAEncoder(m.state_dict())
        cfg = enc.config()
        assert len(ordered_tensors(enc.sd, enc.arch)) == _lib.load().fs2_ecapa_n_tensors(C.byref(cfg))


def test_input_checks_before_any_launch():
    enc = ECAPAEncoder(small().state_dict())
    with pytest.raises(ValueError, match="non-empty"):
        enc(torch.zeros(0, 1000), torch.zeros(0, dtype=torch.int64))
    with pytest.raises(ValueError, match="float32"):
        enc(torch.zeros(2, 1000, dtype=torch.float64), torch.tensor([1000, 1000]))
    with pytest.raises(ValueError, match="lens must be a"):
        enc(torch.zeros(2, 1000), torch.tensor([1000]))
    with pytest.raises(ValueError, match="integer"):
        enc(torch.zeros(2, 1000), torch.tensor([1000.0, 1000.0]))
    with pytest.raises(ValueError, match="CUDA"):
        enc(torch.zeros(2, 1000), torch.tensor([1000, 1000]))
    with pytest.raises(ValueError, match="normalize"):
        enc.encode_batch(torch.zeros(2, 1000), normalize=True)


def test_size_limits():
    enc = ECAPAEncoder(small().state_dict(), "fp32")
    with pytest.raises(ValueError, match="65535"):
        enc.check_size(70000, 16000 * 10)
    enc = ECAPAEncoder(small().state_dict(), "3xf16")
    with pytest.raises(ValueError, match="2\\^31"):
        enc.check_size(1 << 16, 16000 * 300)
    enc.check_size(64, 16000 * 10)


def test_c_entries_refuse_bad_arguments():
    lib = _lib.load()
    cfg = ECAPAEncoder(small().state_dict()).config()
    h = C.c_void_p()
    assert lib.fs2_ecapa_create(C.byref(h), 7, C.byref(cfg)) == -1          # FS2_ERR_INVALID
    cfg.channels = 200
    assert lib.fs2_ecapa_create(C.byref(h), 2, C.byref(cfg)) != 0
    assert b"multiple of 16" in lib.fs2_last_error()


def test_ecapa_kernels_do_not_spill():
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "ecapa.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    lines = open(reports[0]).read().splitlines()
    kernels = [ln for ln in lines if "Compiling entry function" in ln]
    assert len(kernels) >= 15
    for i, ln in enumerate(lines):
        if "Compiling entry function" in ln:
            assert "0 bytes spill stores, 0 bytes spill loads" in lines[i + 2], (ln, lines[i + 2])
