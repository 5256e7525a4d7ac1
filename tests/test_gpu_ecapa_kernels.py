"""Each stage of the ECAPA-TDNN encoder against float64 through fs2_op_ecapa_stage (DESIGN.md section 28): the front end
with digital silence (the -100 dB floor and the top-db clamp bind), block 0's reflected k = 5 convolution, the three
SE-Res2Net blocks (k = 3 at d = 2, 3, 4) on utterances of exactly 5 frames and of lengths that are not multiples of 16,
the MFA, and the attentive statistics pooling with a peaked attention and NaN in masked frames.  Needs an H100."""
import json

import pytest
import torch

from fastspeech2_b200.ecapa import ECAPAEncoder
from oracle import ecapa_oracle as EO
import _ecapa_common as E

pytestmark = pytest.mark.gpu
GATE = {"fp32": 1e-4, "3xf16": 1e-4, "tf32": 2e-2, "f16": 2e-2}
FRAME_LENS = (5, 21, 37)


def stacked(xs, L, nan=True):
    """[T_b, W] float64 tensors -> fp32 rows [B * L, W] on the GPU, NaN past each length."""
    W = xs[0].shape[1]
    out = torch.full((len(xs), L, W), float("nan") if nan else 0.0, dtype=torch.float32, device="cuda")
    for b, x in enumerate(xs):
        out[b, : x.shape[0]] = x.float()
    return out.reshape(len(xs) * L, W)


def check(name, mode, got, want):
    err = max(float((g.double() - w).abs().max() / w.abs().max()) for g, w in zip(got, want))
    print(json.dumps({"stage": name, "mode": mode, "max_abs_over_max": err}))
    assert err <= GATE[mode], (name, mode, err)


@pytest.fixture(scope="module")
def inter():
    """float64 intermediates of three utterances of 5, 21 and 37 frames: features, block outputs, MFA output."""
    m = E.model(512)
    g = torch.Generator().manual_seed(3)
    wavs = [0.2 * torch.randn((n - 1) * 160 + 17, generator=g) for n in FRAME_LENS]
    m.double()
    with torch.no_grad():
        feats = [EO.features(w.cuda().double()) for w in wavs]
        xs = [[f.t()] for f in feats]
        for x in xs:
            for blk in m.blocks:
                x.append(blk(x[-1]))
        mfa = [m.mfa(torch.cat(x[2:], 0)) for x in xs]
    m.float()
    return m, wavs, feats, xs, mfa


@pytest.mark.parametrize("mode", E.MODES)
def test_front_end_with_digital_silence(mode):
    m = E.model(512)
    enc = ECAPAEncoder(m.state_dict(), mode)
    wavs = [E.audio()[5], torch.zeros(1600), E.audio()[3]]
    x, n = E.padded(wavs, nan=True)
    L = x.shape[1]
    T = 1 + L // 160
    got = enc.stage(0, x, n, L, 80, len(wavs) * T).reshape(len(wavs), T, 80)
    for b, w in enumerate(wavs):
        want = EO.features(w.cuda().double())
        err = float((got[b, : want.shape[0]].double() - want).abs().max())
        print(json.dumps({"stage": "front_end", "mode": mode, "b": b, "max_abs_db": err}))
        assert err <= 2e-3, (b, err)


@pytest.mark.parametrize("mode", E.MODES)
def test_block0_reflected_k5(mode, inter):
    m, _, feats, xs, _ = inter
    L = 40
    lens = torch.tensor(FRAME_LENS, device="cuda")
    got = ECAPAEncoder(m.state_dict(), mode).stage(1, stacked(feats, L), lens, L, 512, 3 * L).reshape(3, L, 512)
    check("block0", mode, [got[b, :n] for b, n in enumerate(FRAME_LENS)], [xs[b][1].t() for b in range(3)])


@pytest.mark.parametrize("mode", E.MODES)
@pytest.mark.parametrize("i", [1, 2, 3])
def test_se_res2net_block(mode, i, inter):
    """Block i has k = 3 at dilation i + 1; 5 frames is the shortest length one reflection serves at d = 4."""
    m, _, _, xs, _ = inter
    L = 37
    lens = torch.tensor(FRAME_LENS, device="cuda")
    got = ECAPAEncoder(m.state_dict(), mode).stage(1 + i, stacked([x[i].t() for x in xs], L), lens, L, 512, 3 * L).reshape(3, L, 512)
    check(f"block{i}", mode, [got[b, :n] for b, n in enumerate(FRAME_LENS)], [xs[b][i + 1].t() for b in range(3)])


@pytest.mark.parametrize("mode", E.MODES)
def test_mfa(mode, inter):
    m, _, _, xs, mfa = inter
    L = 48
    lens = torch.tensor(FRAME_LENS, device="cuda")
    x = stacked([torch.cat(x[2:], 0).t() for x in xs], L)
    got = ECAPAEncoder(m.state_dict(), mode).stage(5, x, lens, L, 1536, 3 * L).reshape(3, L, 1536)
    check("mfa", mode, [got[b, :n] for b, n in enumerate(FRAME_LENS)], [h.t() for h in mfa])


@pytest.mark.parametrize("mode", E.MODES)
@pytest.mark.parametrize("peak", [1.0, 30.0])
def test_asp_pooling(mode, peak, inter):
    """peak scales asp.conv, so that the attention is nearly one-hot; frames past each length hold NaN."""
    m, _, _, _, mfa = inter
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    sd["asp.conv.conv.weight"] *= peak
    ref = EO.seeded(0, channels=(512, 512, 512, 512, 1536)).cuda()
    ref.load_state_dict(sd)
    ref.double()
    with torch.no_grad():
        want = [ref.asp(h) for h in mfa]
    L = 40
    lens = torch.tensor(FRAME_LENS, device="cuda")
    got = ECAPAEncoder(sd, mode).stage(6, stacked([h.t() for h in mfa], L), lens, L, 3072, 3)
    check(f"asp_peak{peak:g}", mode, list(got), want)
