"""Synthesis replayed from a CUDA graph at a frame capacity (`graphed_synthesize`, fs2_length_plan_cap): the capacity plan
agrees with fs2_length_plan_ex, every slot that ran is bit-identical to `synthesize` on that utterance alone in every
precision, with and without controls, empty and overflowed slots are +0, replays do not leak rows, the vocoder in the
graph matches the eager vocoder, and the status word raises what `synthesize` raises.  Needs an H100: run with `-m gpu`."""
import pytest
import torch

from fastspeech2_b200 import _lib
from fastspeech2_b200.hifigan import HiFiGANVocoder
from fastspeech2_b200.melgan import MelGANVocoder
from test_gpu_parity import PRECISIONS
from test_gpu_per_utterance import ILENS, build, ragged

pytestmark = pytest.mark.gpu
CAP = 1800            # the seed-7 checkpoint predicts at most 1702 frames for ILENS


@pytest.fixture(scope="module")
def models(weights):
    return {prec: build(weights, prec) for prec in PRECISIONS}


@pytest.fixture(scope="module")
def graphs(models):
    return {prec: models[prec].graphed_synthesize(len(ILENS), max(ILENS), CAP) for prec in PRECISIONS}


def _plans(d_int, il, speed, Lc):
    """(need, cum, d_used) of the capacity plan, and (olens, cum, d_used) of fs2_length_plan_ex, on the same inputs."""
    lib, P = _lib.load(), _lib.ptr
    B, T = d_int.shape
    st = _lib.stream_ptr(d_int.device)
    dev = dict(device="cuda")
    cum_c, cum_e = torch.empty(B, T, dtype=torch.int32, **dev), torch.empty(B, T, dtype=torch.int32, **dev)
    du_c, du_e = torch.empty(B, T, dtype=torch.int64, **dev), torch.empty(B, T, dtype=torch.int64, **dev)
    need, ol_c, ol_e = (torch.empty(B, dtype=torch.int64, **dev) for _ in range(3))
    stats, status = torch.empty(2, dtype=torch.int64, **dev), torch.empty(1, dtype=torch.int32, **dev)
    _lib.check(lib.fs2_length_plan_cap(P(d_int), _lib.FS2_DUR_I64, P(il), P(speed), None, B, T, Lc, P(cum_c), P(ol_c), P(need),
                                       P(du_c), P(status), st), "fs2_length_plan_cap")
    _lib.check(lib.fs2_length_plan_ex(P(d_int), _lib.FS2_DUR_I64, P(il), 1.0, P(speed), B, T, 0, P(cum_e), P(ol_e), P(stats),
                                      P(du_e), st), "fs2_length_plan_ex")
    return (need, ol_c, cum_c, du_c, int(status)), (ol_e, cum_e, du_e)


@pytest.mark.parametrize("per_phoneme_speed", [False, True])
def test_cap_plan_matches_plan_ex(per_phoneme_speed):
    g = torch.Generator().manual_seed(3)
    il = torch.tensor([5, 300, 1, 77, 256, 257, 12, 300])
    B, T = len(il), int(il.max())
    d = torch.randint(0, 40, (B, T), generator=g)
    d[3] = 0                                         # all-zero rule
    for b, n in enumerate(il.tolist()):
        d[b, n:] = 0
    speed = (0.5 + torch.rand(B, T, generator=g)).cuda() if per_phoneme_speed else None
    (need, ol_c, cum_c, du_c, status), (ol_e, cum_e, du_e) = _plans(d.cuda(), il.cuda(), speed, 1 << 20)
    assert status == 0
    assert torch.equal(need, ol_e) and torch.equal(ol_c, ol_e)
    assert torch.equal(cum_c, cum_e) and torch.equal(du_c, du_e)
    # a capacity below some needs: those slots get olens 0 and zero cum / d_used rows, the rest is unchanged
    Lc = int(ol_e.float().median())
    (need, ol_c, cum_c, du_c, status), _ = _plans(d.cuda(), il.cuda(), speed, Lc)
    over = ol_e > Lc
    assert status == _lib.FS2_PLAN_OVERFLOW and torch.equal(need, ol_e)
    assert torch.equal(ol_c, torch.where(over, 0, ol_e))
    assert not cum_c[over].any() and not du_c[over].any()
    assert torch.equal(cum_c[~over], cum_e[~over]) and torch.equal(du_c[~over], du_e[~over])


def _check_slots(out, want, b_of_slot, CAPACITY=CAP):
    """Slot s ran utterance b_of_slot[s] (None: empty): bit-identical to `want[b]`, +0 elsewhere, no NaN anywhere."""
    mels, olens, dur = out[:3]
    assert mels.shape[1] == CAPACITY
    assert not any(torch.isnan(t).any() for t in out if t.dtype.is_floating_point)
    for s, b in enumerate(b_of_slot):
        if b is None:
            assert int(olens[s]) == 0 and not dur[s].any()
            assert not mels[s].any() and not torch.signbit(mels[s]).any()
            continue
        w_mel, w_ol, w_dur = want[b]
        L, n = int(w_ol), w_dur.shape[0]
        assert int(olens[s]) == L, (s, int(olens[s]), L)
        assert torch.equal(dur[s, :n], w_dur) and not dur[s, n:].any(), s
        assert torch.equal(mels[s, :L], w_mel[:L]), f"slot {s}: max diff {(mels[s, :L] - w_mel[:L]).abs().max():.3e}"
        assert not mels[s, L:].any() and not torch.signbit(mels[s, L:]).any(), s


def _alone(m, xs, il, **ctl):
    """synthesize on each utterance alone (B = 1), with its slice of the controls."""
    out = []
    for b, n in enumerate(il.tolist()):
        c = {k: (v[b:b + 1, :n] if v.dim() == 2 else v[b:b + 1]) if torch.is_tensor(v) else v for k, v in ctl.items()}
        with torch.no_grad():
            mels, olens, dur = m.synthesize(xs[b:b + 1, :n].cuda(), il[b:b + 1].cuda(), **c)
        out.append((mels[0], olens[0], dur[0, :n]))
    return out


def _controls(kind, B, T):
    g = torch.Generator().manual_seed(5)
    if kind == "none":
        return {}
    if kind == "scalar":
        return {"speed": 1.3, "pitch": 2.0 ** (3 / 12), "energy": 0.8}
    if kind == "per_utterance":
        return {"speed": 0.7 + torch.rand(B, generator=g), "pitch": 2.0 ** (torch.randint(-6, 7, (B,), generator=g).float() / 12),
                "energy": 0.5 + torch.rand(B, generator=g)}
    return {"speed": 0.6 + torch.rand(B, T, generator=g), "pitch": 0.8 + 0.4 * torch.rand(B, T, generator=g),
            "energy": 0.5 + torch.rand(B, T, generator=g)}


@pytest.mark.parametrize("prec", PRECISIONS)
@pytest.mark.parametrize("kind", ["none", "scalar", "per_utterance", "per_phoneme"])
def test_slots_bit_identical_to_synthesize_alone(models, graphs, prec, kind):
    m, gs = models[prec], graphs[prec]
    xs, il = ragged(ILENS)
    ctl = _controls(kind, *xs.shape)
    want = _alone(m, xs, il, **ctl)
    ran = [b for b in range(len(ILENS)) if int(want[b][1]) <= CAP]
    ctl_dev = {k: v.cuda() if torch.is_tensor(v) else v for k, v in ctl.items()}
    with torch.no_grad():
        out = gs(xs.cuda(), il.cuda(), **ctl_dev)
    torch.cuda.synchronize()
    over = gs.overflowed()
    assert over == [b for b in range(len(ILENS)) if b not in ran]
    assert [int(v) for v in gs.need] == [int(w[1]) for w in want]
    _check_slots(out, want, [b if b in ran else None for b in range(len(ILENS))])


def test_fewer_requests_empty_slots_and_no_stale_rows(models, graphs):
    m, gs = models["3xtf32"], graphs["3xtf32"]
    xs, il = ragged(ILENS)
    want = _alone(m, xs, il)
    with torch.no_grad():
        gs(xs.cuda(), il.cuda())
        sub = [4, 1, 6]                               # a second, shorter request: 3 slots of at most 100 phonemes
        t = max(ILENS[b] for b in sub)
        out = gs(xs[sub, :t], il[sub])                # host tensors are accepted too
    _check_slots(out, want, sub + [None] * (len(ILENS) - len(sub)))
    with torch.no_grad():                             # an explicitly empty slot among real ones
        il0 = il[sub].clone()
        il0[1] = 0
        out = gs(xs[sub, :t].cuda(), il0.cuda())
    _check_slots(out, want, [4, None, 6] + [None] * (len(ILENS) - len(sub)))


def test_overflow_is_reported_not_raised(models):
    m = models["3xtf32"]
    xs, il = ragged(ILENS)
    want = _alone(m, xs, il)
    cap = sorted(int(w[1]) for w in want)[4]          # half the utterances do not fit
    gs = m.graphed_synthesize(len(ILENS), max(ILENS), cap)
    with torch.no_grad():
        out = gs(xs.cuda(), il.cuda())
    over = [b for b in range(len(ILENS)) if int(want[b][1]) > cap]
    assert over and gs.overflowed() == over
    assert all(int(gs.need[b]) == int(want[b][1]) for b in over)
    _check_slots(out, want, [None if b in over else b for b in range(len(ILENS))], cap)


@pytest.mark.parametrize("name", ["hifigan_v3", "melgan"])
def test_vocoder_in_the_graph_matches_the_eager_vocoder(models, name):
    m = models["3xtf32"]
    torch.manual_seed(0)
    v = (HiFiGANVocoder("v3") if name == "hifigan_v3" else MelGANVocoder()).cuda()
    xs, il = ragged(ILENS[:4])
    gs = m.graphed_synthesize(6, max(ILENS), CAP, vocoder=v)
    with torch.no_grad():
        mels_e, olens_e, _ = m.synthesize(xs.cuda(), il.cuda())
        mels, olens, dur, audio, alens = gs(xs.cuda(), il.cuda())
        assert torch.equal(alens, olens * 256) and torch.equal(olens[:4], olens_e)
        for b in range(4):
            L = int(olens[b])
            one, _ = v(mels_e[b:b + 1, :L].contiguous(), olens_e[b:b + 1])
            assert torch.equal(audio[b, :L * 256], one[0]), b
            assert not audio[b, L * 256:].any()
        assert not audio[4:].any() and not alens[4:].any()
    assert torch.isfinite(audio).all()


def test_bad_ilens_and_bad_factors_raise(models, graphs):
    gs = graphs["3xtf32"]
    xs, il = ragged(ILENS)
    bad = il.clone()
    bad[2] = max(ILENS) + 1
    with pytest.raises(ValueError, match="ilens"):
        gs(xs.cuda(), bad.cuda())
    speed = torch.ones(xs.shape)
    speed[3, 5] = 0.0
    with pytest.raises(ValueError, match="non-finite or <= 0"):
        gs(xs.cuda(), il.cuda(), speed=speed.cuda())
    with pytest.raises(ValueError, match="non-finite or <= 0"):
        gs(xs.cuda(), il.cuda(), pitch=torch.full((len(ILENS),), float("nan")).cuda())
    # deferred: the call returns, the next call (or flush) raises
    gs(xs.cuda(), bad.cuda(), validate="deferred")
    with pytest.raises(ValueError, match="ilens"):
        gs(xs.cuda(), il.cuda(), validate="deferred")
    gs.flush()                                        # the raise consumed the pending check: nothing is left
    gs(xs.cuda(), il.cuda(), speed=speed.cuda(), validate="deferred")
    with pytest.raises(ValueError, match="non-finite or <= 0"):
        gs.flush()
    gs(xs.cuda(), bad.cuda(), validate=False)         # no check at all
    gs.flush()


def test_parameter_update_after_capture_raises(weights):
    m = build(weights, "3xf16")
    gs = m.graphed_synthesize(2, 40, 600)
    xs, il = ragged([40, 12])
    with torch.no_grad():
        gs(xs.cuda(), il.cuda())
        m.feat_out.bias.add_(1.0)
    with pytest.raises(RuntimeError, match="parameters changed since capture"):
        gs(xs.cuda(), il.cuda())
