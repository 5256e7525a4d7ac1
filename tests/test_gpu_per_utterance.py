"""Per-utterance batching (`synthesize`, `_forward(..., per_utterance=True)`): an utterance's result is bit-identical to
the same utterance run alone (B = 1), whatever else is in its batch, in every precision mode, and every padded position
of every returned tensor is exactly 0.  Bit-identity, not a tolerance: durations are integers and would flip.
Needs an H100: run with `-m gpu`."""
import pytest
import torch

from fastspeech2_b200 import FeedForwardTransformer
from fastspeech2_b200.hparams import load_hp
from fastspeech2_b200.serving import export_torchscript
from fastspeech2_b200.synthetic import make_batch
from oracle import fs2_oracle as O
from test_gpu_parity import PRECISIONS, TOL, close

pytestmark = pytest.mark.gpu
T_ = torch.from_numpy
# 1 phoneme up to > 128, the longest not in row 0; the seed-7 checkpoint predicts 10 .. 1702 frames for these
ILENS = [37, 1, 150, 64, 9, 129, 100, 17]


def ragged(ilens, seed=21):
    g = torch.Generator().manual_seed(seed)
    xs = torch.zeros(len(ilens), max(ilens), dtype=torch.int64)
    for b, n in enumerate(ilens):
        xs[b, :n] = torch.randint(1, 68, (n,), generator=g)
    return xs, torch.tensor(ilens)


def build(sd, prec):
    m = FeedForwardTransformer(68, 80, load_hp(), precision=prec)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


@pytest.fixture(scope="module")
def models(weights):
    return {prec: build(weights, prec) for prec in PRECISIONS}


def check_synthesize(m, xs, il):
    """synthesize on the batch == inference / B = 1 _forward per utterance, bit for bit; zeros past the lengths."""
    with torch.no_grad():
        mels, olens, dur = m.synthesize(xs.cuda(), il.cuda())
    assert olens.dtype == torch.int64 and dur.dtype == torch.int64 and mels.shape[1] == int(olens.max())
    for b, n in enumerate(il.tolist()):
        with torch.no_grad():
            want = m.inference(xs[b, :n].cuda())
            _, _, d1, _, _ = m._forward(xs[b:b + 1, :n].cuda(), il[b:b + 1].cuda(), is_inference=True, _one_hot=False)
        L = int(olens[b])
        assert want.shape[0] == L, (b, want.shape, L)
        assert torch.equal(dur[b, :n], d1[0]) and not dur[b, n:].any(), f"durations of utterance {b}"
        assert torch.equal(mels[b, :L], want), f"mels of utterance {b}: max diff {(mels[b, :L] - want).abs().max():.3e}"
        assert not mels[b, L:].any(), f"padded frames of utterance {b}"
    return mels, olens, dur


@pytest.mark.parametrize("prec", PRECISIONS)
def test_synthesize_bit_identical_to_single_utterance(models, prec):
    m = models[prec]
    xs, il = ragged(ILENS)
    mels, olens, dur = check_synthesize(m, xs, il)
    ol = olens.cpu()
    # the lengths cross several 128-row tiles, and some utterances end inside the first one (dead tiles behind them)
    assert int(ol.max()) > 3 * 128 and int(ol.min()) < 128 and int(ol.argmax()) != 0, ol.tolist()
    # the same utterances in the reverse order: nothing changes for any of them
    with torch.no_grad():
        mels_r, olens_r, dur_r = m.synthesize(xs.flip(0).cuda(), il.flip(0).cuda())
    B = len(ILENS)
    for b in range(B):
        L, r = int(ol[b]), B - 1 - b
        assert int(olens_r[r]) == L and torch.equal(dur_r[r], dur[b]) and torch.equal(mels_r[r, :L], mels[b, :L])
    # the 5-tuple of _forward: one-hot rows of padded frames are all-zero, valid frames match the B = 1 call
    with torch.no_grad():
        before, after, d, oh_e, oh_p = m._forward(xs.cuda(), il.cuda(), is_inference=True, per_utterance=True)
    assert torch.equal(after, mels) and torch.equal(d, dur)
    for b, n in enumerate(ILENS):
        L = int(ol[b])
        with torch.no_grad():
            b1, _, _, e1, p1 = m._forward(xs[b:b + 1, :n].cuda(), il[b:b + 1], is_inference=True)
        assert torch.equal(before[b, :L], b1[0]) and torch.equal(oh_e[b, :L], e1[0]) and torch.equal(oh_p[b, :L], p1[0])
        assert not before[b, L:].any() and not oh_e[b, L:].any() and not oh_p[b, L:].any()


@pytest.mark.parametrize("prec", PRECISIONS)
def test_synthesize_all_zero_durations(weights, prec):
    """A duration head that predicts 0 everywhere: the all-ones rule fires per utterance (olens == ilens; like the
    reference's in-place fill_, the returned durations read 1 there)."""
    sd = {k: v.clone() for k, v in weights.items()}
    sd["duration_predictor.linear.weight"].zero_()
    sd["duration_predictor.linear.bias"].fill_(-20.0)          # round(exp(-20) - 1) = 0
    m = build(sd, prec)
    xs, il = ragged(ILENS, seed=3)
    _, olens, dur = check_synthesize(m, xs, il)
    ones = (torch.arange(xs.shape[1])[None, :] < il[:, None]).long()
    assert torch.equal(olens.cpu(), il) and torch.equal(dur.cpu(), ones)


@pytest.mark.parametrize("prec", PRECISIONS)
def test_teacher_forced_per_utterance_filelist(models, golden, prec):
    """Real LJSpeech lengths (first 64 rows of the filelist, olens 222 .. 856)."""
    from _synth import seeded_energy_pitch
    g = golden("filelist64")
    olens = T_(g["olens"])
    es, ps = seeded_energy_pitch(int(g["es_seed"]), olens, int(olens.max()))
    check_teacher_forced(models[prec], T_(g["xs"]), T_(g["ilens"]), olens, T_(g["ds"]), es, ps)


@pytest.mark.parametrize("prec", PRECISIONS)
def test_teacher_forced_per_utterance_tile_edges(models, prec):
    """Lengths on and around the 16-row granule and the 128-row tile, where the packed-tail and dead-tile logic changes."""
    bt = make_batch(7, 129, 300, seed=77, ilens=[5, 16, 17, 40, 128, 129, 70], olens=[15, 16, 17, 127, 128, 129, 300])
    check_teacher_forced(models[prec], bt["xs"], bt["ilens"], bt["olens"], bt["ds"], bt["es"], bt["ps"])


def check_teacher_forced(m, xs, il, ol, ds, es, ps):
    with torch.no_grad():
        got = m._forward(xs.cuda(), il.cuda(), ol.cuda(), ds.cuda(), es.cuda(), ps.cuda(), per_utterance=True)
    for b, (n, L) in enumerate(zip(il.tolist(), ol.tolist())):
        with torch.no_grad():
            want = m._forward(xs[b:b + 1, :n].cuda(), il[b:b + 1].cuda(), ol[b:b + 1].cuda(), ds[b:b + 1, :n].cuda(),
                              es[b:b + 1, :L].cuda(), ps[b:b + 1, :L].cuda())
        for name, gt, wt, k in zip(("before", "after", "d_outs", "e_outs", "p_outs"), got, want, (L, L, n, L, L)):
            assert torch.equal(gt[b, :k], wt[0]), f"{name} of utterance {b} (ilen {n}, olen {L})"
            assert not gt[b, k:].any(), f"padded {name} of utterance {b}"


@pytest.mark.parametrize("prec", PRECISIONS)
def test_synthesize_against_oracle(models, weights, prec):
    """synthesize against the CPU oracle run on the utterance alone: durations and bucket ids exact, mels within TOL."""
    m = models[prec]
    xs, il = ragged(ILENS)
    with torch.no_grad():
        _, after, d, oh_e, oh_p = m._forward(xs.cuda(), il.cuda(), is_inference=True, per_utterance=True)
    for b in (1, 4, 0):
        n = ILENS[b]
        w_before, w_after, w_d, w_e, w_p = O.forward_path(weights, xs[b:b + 1, :n], il[b:b + 1], is_inference=True)
        L = w_after.shape[1]
        assert torch.equal(d[b, :n].cpu(), w_d[0].long()) and not d[b, n:].any()
        assert not after[b, L:].any()
        assert torch.equal(oh_e[b, :L].argmax(-1).cpu(), w_e[0].argmax(-1))
        assert torch.equal(oh_p[b, :L].argmax(-1).cpu(), w_p[0].argmax(-1))
        close(after[b, :L], w_after[0], TOL[prec], f"after of utterance {b} ({prec})")


def test_served_synthesize_matches_model(tmp_path, models):
    m = models["3xtf32"]
    served = torch.jit.load(export_torchscript(m, str(tmp_path / "fs2.pt"))).cuda()
    xs, il = ragged(ILENS)
    with torch.no_grad():
        want, want_ol, _ = m.synthesize(xs.cuda(), il.cuda())
    got, got_ol = served.synthesize(xs.cuda(), il.cuda())
    assert torch.equal(got, want) and torch.equal(got_ol, want_ol)
