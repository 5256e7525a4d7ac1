"""The ECAPA-TDNN speaker encoder on the GPU (DESIGN.md section 28): the embedding against a float64 oracle in every math
mode, bit identity across batches, NaN past the lengths, repeated calls, graph replay and sign, gain invariance, the
operand-plane range error, and the `speakers embed` -> `average` -> `synthesize(spembs=)` pipeline.  Weights are seeded,
the BatchNorm statistics come from a float64 pass over the test audio.  Needs an H100: run with `-m gpu`."""
import json
import os

import numpy as np
import pytest
import torch

from fastspeech2_b200.ecapa import ECAPAEncoder
import _ecapa_common as E

pytestmark = pytest.mark.gpu
GATE = {"fp32": 1e-3, "3xf16": 1e-3, "tf32": 5e-2, "f16": 5e-2}   # max-abs error over max |e|


def rel_err(got, want):
    return float((got.double() - want).abs().max() / want.abs().max())


def cosine(got, want):
    return float(torch.nn.functional.cosine_similarity(got.double(), want, dim=0))


def test_embedding_matches_float64_oracle_in_every_mode():
    m = E.model()
    wavs = E.audio()
    want = [E.reference(m, w) for w in wavs]
    x, n = E.padded(wavs)
    errs = {}
    for mode in E.MODES:
        got = ECAPAEncoder(m.state_dict(), mode)(x, n)
        errs[mode] = max(rel_err(got[b], want[b]) for b in range(len(wavs)))
        cos = min(cosine(got[b], want[b]) for b in range(len(wavs)))
        print(json.dumps({"mode": mode, "max_abs_over_max": errs[mode], "min_cosine": cos}))
        assert errs[mode] <= GATE[mode], (mode, errs[mode])
        assert cos > 0.999, (mode, cos)
    # the fp32-class modes must beat the single-plane ones, so a lost lo plane fails
    assert max(errs["fp32"], errs["3xf16"]) < min(errs["f16"], errs["tf32"]), errs


def test_global_context_fold_rounding_is_recorded():
    m = E.model()
    w = E.audio()[2].cuda().double()
    with torch.no_grad():
        m.double()
        a, b = m.embed(w), m.embed(w, fold=True)
        m.float()
    d = rel_err(b, a)
    print(json.dumps({"fold_vs_unfolded_float64": d}))
    assert d < 1e-12


@pytest.mark.parametrize("mode", E.MODES)
def test_batch_is_bit_identical_to_each_utterance_alone(mode):
    m = E.model(512)
    enc = ECAPAEncoder(m.state_dict(), mode)
    wavs = E.audio()
    x, n = E.padded(wavs)
    got = enc(x, n)
    for b, w in enumerate(wavs):
        alone = enc(w[None].cuda(), torch.tensor([len(w)], device="cuda"))
        assert torch.equal(alone[0], got[b]), (mode, b)
    xr, nr = E.padded(wavs[::-1])
    assert torch.equal(enc(xr, nr).flip(0), got)
    xn, nn_ = E.padded(wavs, nan=True)
    assert torch.equal(enc(xn, nn_), got)                          # samples past lens are never read
    assert torch.equal(enc(x, n), got) and torch.equal(enc(x, n), got)
    assert torch.equal(enc(-x, n), got)                            # the power spectrum is even in x


def test_graph_replay_equals_eager_call():
    enc = ECAPAEncoder(E.model(512).state_dict(), "3xf16")
    x, n = E.padded(E.audio())
    eager = enc(x, n)
    from fastspeech2_b200 import _lib
    from fastspeech2_b200._kernel_module import query_bytes, workspace
    h = enc._handle(x.device)
    ws = workspace(enc._ws, x.device, query_bytes("fs2_ecapa_workspace_bytes", h, x.shape[0], x.shape[1]))
    emb = torch.empty_like(eager)
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            _lib.check(_lib.load().fs2_ecapa(h, x.data_ptr(), n.data_ptr(), x.shape[0], x.shape[1], emb.data_ptr(), status.data_ptr(),
                                             ws.data_ptr(), ws.numel(), s.cuda_stream), "fs2_ecapa")
    emb.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    assert torch.equal(emb, eager)


def test_gain_invariance():
    """Mean normalisation cancels the 20 log10(0.5) dB shift, so 0.5 x matches x within the fp32-class gate."""
    enc = ECAPAEncoder(E.model(512).state_dict(), "fp32")
    wavs = E.audio()[:5]                          # no digital silence: the -100 dB floor does not shift
    x, n = E.padded(wavs)
    a, b = enc(x, n), enc(0.5 * x, n)
    err = max(rel_err(b[i], a[i].double()) for i in range(len(wavs)))
    print(json.dumps({"gain_0.5_max_abs_over_max": err}))
    assert err <= GATE["fp32"]


def test_scaled_weight_raises_range_error_in_plane_modes_only():
    sd = {k: v.clone() for k, v in E.model(512).state_dict().items()}
    sd["blocks.1.tdnn1.conv.conv.weight"] *= 1e5
    x, n = E.padded(E.audio()[:2])
    for mode in ("f16", "3xf16"):
        with pytest.raises(ValueError, match="operand planes"):
            ECAPAEncoder(sd, mode)(x, n)
    assert torch.isfinite(ECAPAEncoder(sd, "fp32")(x, n)).all()


def test_short_utterance_on_the_device_is_a_value_error():
    enc = ECAPAEncoder(E.model(512).state_dict(), "3xf16")
    x, _ = E.padded(E.audio()[:2])
    with pytest.raises(ValueError, match="lens"):
        enc(x, torch.tensor([639, x.shape[1]], device="cuda"))


def test_encode_batch_relative_lengths():
    enc = ECAPAEncoder(E.model(512).state_dict(), "3xf16")
    wavs = E.audio()[2:4]
    x, n = E.padded(wavs)
    got = enc.encode_batch(x, n.double() / x.shape[1])
    assert got.shape == (2, 1, enc.dim)
    assert torch.equal(got[:, 0], enc(x, n))
    with pytest.raises(ValueError, match="normalize"):
        enc.encode_batch(x, normalize=True)


def test_speakers_embed_average_and_synthesize(tmp_path):
    from scipy.io import wavfile

    from fastspeech2_b200 import FeedForwardTransformer, synthetic_state_dict
    from fastspeech2_b200.data import load_spemb
    from fastspeech2_b200.hparams import load_hp
    from fastspeech2_b200.speakers import average, main
    m = E.model(512)
    ck = tmp_path / "embedding_model.ckpt"
    torch.save(m.state_dict(), ck)
    wd = tmp_path / "wavs"
    wd.mkdir()
    g = np.random.default_rng(1)
    names = ["spkA_001", "spkA_002", "spkB_001"]
    for i, nm in enumerate(names):
        sr = 22050 if i == 0 else 16000
        wavfile.write(str(wd / f"{nm}.wav"), sr, (g.standard_normal(sr + 500 * i) * 3000).astype(np.int16))
    out = tmp_path / "spemb"
    main(["embed", "--checkpoint", str(ck), "-d", str(wd), "-o", str(out), "--math-mode", "3xf16"])
    es = {nm: load_spemb(str(out / f"{nm}.npy")) for nm in names}
    assert all(e.shape == (192,) and e.dtype == np.float32 and np.isfinite(e).all() for e in es.values())
    fl = tmp_path / "filelist.txt"
    fl.write_text("".join(f"text|1 2|1 1|a b|{nm}.wav\n" for nm in names))
    means = average(str(fl), str(out))
    assert sorted(means) == ["spkA", "spkB"]
    hp = load_hp()
    hp["model"]["spk_embed_dim"] = 192
    fs2 = FeedForwardTransformer(68, 80, hp, precision="3xf16")
    sd = dict(synthetic_state_dict(7))
    gen = torch.Generator().manual_seed(0)
    sd["spk_embed_proj.weight"] = 0.05 * torch.randn(256, 192, generator=gen)
    sd["spk_embed_proj.bias"] = torch.zeros(256)
    fs2.load_state_dict(sd, strict=True)
    fs2 = fs2.cuda().eval()
    enc = ECAPAEncoder(m.state_dict(), "3xf16")
    x, n = E.padded(E.audio()[2:4])
    xs = torch.randint(1, 60, (2, 12), device="cuda")
    xs[1, 9:] = 0
    mels, olens, _ = fs2.synthesize(xs, torch.tensor([12, 9], device="cuda"), spembs=enc(x, n))
    assert torch.isfinite(mels).all() and bool((olens > 0).all())
