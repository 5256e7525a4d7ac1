"""The duration aligner on the H100 (fastspeech2_b200.aligner, csrc/aligner.cu) against the float64 oracle
(oracle/aligner_oracle.py), on ragged batches with T = 1, L = T and L much larger than T; inputs carry NaN past the
lengths and outputs sit between sentinel guard bands, and neither may change a bit.  MAS must match the float32 oracle
bit for bit on the kernel's own logp; every utterance must be bit-identical to its B = 1 call and to the reversed batch;
one training step must match the float64 model; and an aligner trained on a synthetic corpus must recover its durations.

Gates are about 3x the worst value measured on an H100 80GB HBM3 at a 700 W power limit (DESIGN.md section 24):
  logp                max |logp - ref|                          LOGP_GATE
  dq, dk              max |g - ref| / max |ref|                 DQK_GATE
  forward-sum         |loss - ref| / ref, and dlogp as dq       FS_GATE, FS_GRAD_GATE
  bin loss            |loss - ref| / ref, and dlogp as dq       BIN_GATE
  train step          loss rel., each gradient as dq            STEP_LOSS_GATE, STEP_GRAD_GATE (TF32 convolutions)
  recovery            phonemes more than 1 frame off the truth  MISS_GATE"""
import json
import os

import numpy as np
import pytest
import torch

from _aligner_corpus import fixture_lines, render
from conftest import REPO
from fastspeech2_b200 import _lib
from fastspeech2_b200 import aligner as A
from oracle import aligner_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENT = 12345.0
LOGP_GATE = 6e-6            # measured 2.0e-6
DQK_GATE = 1.5e-6           # 4.7e-7
FS_GATE = 3e-7              # 9.4e-8
FS_GRAD_GATE = 2e-5         # 6.8e-6
BIN_GATE = 4e-7             # 1.2e-7 (loss and gradient)
STEP_LOSS_GATE = 3.5e-5     # 1.1e-5
STEP_GRAD_GATE = 0.1        # 3.1e-2: the convolutions' operands are rounded to TF32
MISS_GATE = 0.1             # 0.011; training is not bit-reproducible (atomic embedding and bias gradients), and a run
                            # with binarization from step 750 missed 0.04-0.07 along its way (DESIGN.md section 24)

CASES = {"t1": [(1, 1), (1, 9), (1, 4)],
         "square": [(6, 6), (4, 6), (5, 5), (2, 2)],
         "long": [(3, 240), (17, 400), (9, 150), (12, 12), (30, 333)]}


def _report(name, value):
    print(f"MEASURED {name} {value:.3e}")


def _lens(case):
    N = [n for n, _ in CASES[case]]
    M = [m for _, m in CASES[case]]
    return N, M, max(N) + 2, max(M) + 3


def _qk(case, seed=0):
    """q [B, L, 80], k [B, T, 80] (scale 8) with NaN past the lengths, and the lengths on the device."""
    N, M, T, L = _lens(case)
    g = torch.Generator().manual_seed(seed)
    q = torch.full((len(N), L, 80), float("nan"))
    k = torch.full((len(N), T, 80), float("nan"))
    for b, (n, m) in enumerate(zip(N, M)):
        q[b, :m] = 8 * torch.randn(m, 80, generator=g)
        k[b, :n] = 8 * torch.randn(n, 80, generator=g)
    return q.to(DEV), k.to(DEV), torch.tensor(N, device=DEV), torch.tensor(M, device=DEV)


def _guarded(shape, dtype=torch.float32, sent=SENT):
    """(view of shape, whole buffer): 64 sentinel elements before and after."""
    n = int(np.prod(shape))
    buf = torch.full((n + 128,), sent, dtype=dtype, device=DEV)
    return buf[64: 64 + n].view(shape), buf


def _bands_intact(buf, sent=SENT):
    return bool((buf[:64] == sent).all() and (buf[-64:] == sent).all())


def _ws(B, L, T):
    return torch.empty(A.workspace_bytes(B, L, T), dtype=torch.uint8, device=DEV)


def _logprob(q, k, il, ol):
    B, L, T = q.shape[0], q.shape[1], k.shape[1]
    out, buf = _guarded((B, L, T))
    st = torch.zeros(1, dtype=torch.int32, device=DEV)
    ws = _ws(B, L, T)
    _lib.check(_lib.load().fs2_align_logprob(q.data_ptr(), k.data_ptr(), il.data_ptr(), ol.data_ptr(), B, L, T, out.data_ptr(), st.data_ptr(),
                                             ws.data_ptr(), ws.numel(), _lib.stream_ptr(q.device)), "fs2_align_logprob")
    assert _bands_intact(buf)
    return out, int(st.item())


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("case", list(CASES))
def test_logprob_and_its_gradients_against_float64(case):
    q, k, il, ol = _qk(case)
    B, L, T = q.shape[0], q.shape[1], k.shape[1]
    logp, st = _logprob(q, k, il, ol)
    assert st == 0
    q64 = torch.nan_to_num(q.double().cpu()).requires_grad_(True)
    k64 = torch.nan_to_num(k.double().cpu()).requires_grad_(True)
    ref = O.logprob(q64, k64, il.cpu(), ol.cpu())
    err = float((logp.double().cpu() - ref.detach()).abs().max())
    _report(f"logp[{case}]", err)
    assert err <= LOGP_GATE
    valid = ref.detach() != 0
    assert not logp.cpu()[~valid].any()                                   # +0 outside the lengths
    dl = torch.randn(B, L, T, generator=torch.Generator().manual_seed(1))
    dl_dev = dl.to(DEV).masked_fill(~valid.to(DEV), float("nan"))         # dlogp past the lengths is never read
    ref.backward(dl.double() * valid)
    dq, bq = _guarded((B, L, 80))
    dk, bk = _guarded((B, T, 80))
    st_t = torch.zeros(1, dtype=torch.int32, device=DEV)
    ws = _ws(B, L, T)
    _lib.check(_lib.load().fs2_align_logprob_backward(q.data_ptr(), k.data_ptr(), il.data_ptr(), ol.data_ptr(), B, L, T, dl_dev.data_ptr(),
                                                      dq.data_ptr(), dk.data_ptr(), st_t.data_ptr(), ws.data_ptr(), ws.numel(),
                                                      _lib.stream_ptr(q.device)), "fs2_align_logprob_backward")
    assert _bands_intact(bq) and _bands_intact(bk) and int(st_t.item()) == 0
    eq, ek = _rel(dq, q64.grad), _rel(dk, k64.grad)
    _report(f"dq[{case}]", eq)
    _report(f"dk[{case}]", ek)
    assert eq <= DQK_GATE and ek <= DQK_GATE
    assert torch.isfinite(dq).all() and torch.isfinite(dk).all()


def _forward_sum(logp, il, ol, dloss=None, grad=True):
    B, L, T = logp.shape
    loss, bl = _guarded((B,))
    dlogp, bd = _guarded((B, L, T)) if grad else (None, None)
    st = torch.zeros(1, dtype=torch.int32, device=DEV)
    ws = _ws(B, L, T)
    _lib.check(_lib.load().fs2_align_forward_sum(logp.data_ptr(), il.data_ptr(), ol.data_ptr(), B, L, T, None if dloss is None else dloss.data_ptr(),
                                                 loss.data_ptr(), None if dlogp is None else dlogp.data_ptr(), st.data_ptr(), ws.data_ptr(),
                                                 ws.numel(), _lib.stream_ptr(logp.device)), "fs2_align_forward_sum")
    assert _bands_intact(bl) and (bd is None or _bands_intact(bd))
    return loss, dlogp, int(st.item())


@pytest.mark.parametrize("case", list(CASES))
def test_forward_sum_against_float64_ctc(case):
    q, k, il, ol = _qk(case)
    logp, _ = _logprob(q, k, il, ol)
    B, L, T = logp.shape
    # an infeasible utterance: more phonemes than frames
    il2 = il.clone()
    il2[0] = min(T, int(ol[0]) + 1) if int(ol[0]) + 1 <= T else il[0]
    infeasible = int(il2[0]) > int(ol[0])
    valid = torch.zeros(B, L, T, dtype=torch.bool)
    for b in range(B):
        valid[b, : int(ol[b]), : int(il2[b])] = True
    lp_in = logp.clone().masked_fill(~valid.to(DEV), float("nan"))
    dloss = torch.rand(B, generator=torch.Generator().manual_seed(2)).to(DEV) + 0.5
    loss, dlogp, st = _forward_sum(lp_in, il2, ol, dloss)
    loss_only, none, st2 = _forward_sum(lp_in, il2, ol, grad=False)
    assert torch.equal(loss, loss_only) and st2 == st
    assert st == (_lib.FS2_ALIGN_INFEASIBLE if infeasible else 0)
    lp64 = logp.double().cpu().masked_fill(~valid, 0).requires_grad_(True)
    ref = O.forward_sum(lp64, il2.cpu(), ol.cpu())
    (ref * dloss.double().cpu()).sum().backward()
    e = _rel(loss, ref.detach())
    eg = _rel(dlogp, lp64.grad)
    _report(f"forward_sum[{case}]", e)
    _report(f"forward_sum_grad[{case}]", eg)
    assert e <= FS_GATE and eg <= FS_GRAD_GATE
    assert not dlogp.cpu()[~valid].any()
    if infeasible:
        assert float(loss[0]) == 0 and not dlogp[0].any()


def _mas(logp, il, ol):
    B, L, T = logp.shape
    dur, bd = _guarded((B, T), torch.int64, -7)
    path, bp = _guarded((B, L), torch.int32, -7)
    st = torch.zeros(1, dtype=torch.int32, device=DEV)
    ws = _ws(B, L, T)
    _lib.check(_lib.load().fs2_align_mas(logp.data_ptr(), il.data_ptr(), ol.data_ptr(), B, L, T, dur.data_ptr(), path.data_ptr(), st.data_ptr(),
                                         ws.data_ptr(), ws.numel(), _lib.stream_ptr(logp.device)), "fs2_align_mas")
    assert _bands_intact(bd, -7) and _bands_intact(bp, -7)
    return dur, path, int(st.item())


@pytest.mark.parametrize("case", list(CASES))
def test_mas_is_bit_identical_to_the_float32_oracle(case):
    q, k, il, ol = _qk(case)
    logp, _ = _logprob(q, k, il, ol)
    logp[1, :, :] = 0.0                                  # constant rows: every step of that utterance is a tie
    lp_in = logp.clone()
    for b in range(logp.shape[0]):
        lp_in[b, int(ol[b]):] = float("nan")
        lp_in[b, :, int(il[b]):] = float("nan")
    dur, path, st = _mas(lp_in, il, ol)
    assert st == 0
    rd, rp = O.mas(logp.cpu().numpy(), il.cpu().numpy(), ol.cpu().numpy())
    assert np.array_equal(dur.cpu().numpy(), rd) and np.array_equal(path.cpu().numpy(), rp)
    for b in range(logp.shape[0]):
        d = dur[b, : int(il[b])]
        assert int(d.min()) >= 1 and int(d.sum()) == int(ol[b])


def test_mas_refuses_infeasible_and_bad_lengths():
    q, k, il, ol = _qk("long")
    logp, _ = _logprob(q, k, il, ol)
    il2, ol2 = il.clone(), ol.clone()
    il2[1] = 0
    ol2[2] = 5                                            # 9 phonemes, 5 frames
    dur, path, st = _mas(logp, il2, ol2)
    assert st == _lib.FS2_ALIGN_BAD_LENGTH | _lib.FS2_ALIGN_INFEASIBLE
    for b in (1, 2):
        assert not dur[b].any() and (path[b] == -1).all()
    assert int(dur[0].sum()) == int(ol[0])


@pytest.mark.parametrize("case", list(CASES))
def test_bin_loss_against_float64(case):
    q, k, il, ol = _qk(case)
    logp, _ = _logprob(q, k, il, ol)
    B, L, T = logp.shape
    _, path, _ = _mas(logp, il, ol)
    loss, bl = _guarded((B,))
    dlogp, bd = _guarded((B, L, T))
    st = torch.zeros(1, dtype=torch.int32, device=DEV)
    ws = _ws(B, L, T)
    dloss = torch.rand(B, generator=torch.Generator().manual_seed(4)).to(DEV) + 0.5
    _lib.check(_lib.load().fs2_align_bin_loss(logp.data_ptr(), path.data_ptr(), il.data_ptr(), ol.data_ptr(), B, L, T, dloss.data_ptr(),
                                              loss.data_ptr(), dlogp.data_ptr(), st.data_ptr(), ws.data_ptr(), ws.numel(),
                                              _lib.stream_ptr(logp.device)), "fs2_align_bin_loss")
    assert _bands_intact(bl) and _bands_intact(bd) and int(st.item()) == 0
    lp64 = logp.double().cpu().requires_grad_(True)
    ref = O.bin_loss(lp64, path.cpu().numpy(), il.cpu(), ol.cpu())
    (ref * dloss.double().cpu()).sum().backward()
    e, eg = _rel(loss, ref.detach()), _rel(dlogp, lp64.grad)
    _report(f"bin[{case}]", e)
    _report(f"bin_grad[{case}]", eg)
    assert e <= BIN_GATE and eg <= BIN_GATE


def _model_batch(n, seed):
    lines = fixture_lines(64)[:n]
    sym = A.build_symbols(fixture_lines())
    mels = render(lines, seed)
    corpus = A.Corpus(lines, sym, mels=mels)
    return corpus, sym


def test_durations_are_per_utterance_bit_identical():
    corpus, sym = _model_batch(9, 3)
    torch.manual_seed(0)
    model = A.Aligner(len(sym)).to(DEV)
    idx = list(range(9))
    xs, il, mels, ol = corpus.batch(idx, DEV)
    mels = mels.clone()
    for b in range(9):
        mels[b, int(ol[b]):] = float("nan")              # NaN in the padding changes nothing
    dur, st = model.durations(xs, il, mels, ol)
    assert st == 0
    rx, ri, rm, ro = corpus.batch(idx[::-1], DEV)
    rdur, _ = model.durations(rx, ri, rm, ro)
    for b in range(9):
        x1, i1, m1, o1 = corpus.batch([b], DEV)
        d1, _ = model.durations(x1, i1, m1, o1)
        n = int(il[b])
        assert torch.equal(dur[b, :n], d1[0]) and torch.equal(rdur[8 - b, :n], d1[0])
        assert not dur[b, n:].any() and int(dur[b].sum()) == int(ol[b]) and int(dur[b, :n].min()) >= 1


def test_train_step_against_the_float64_model_and_three_steps_lower_the_loss():
    corpus, sym = _model_batch(6, 5)
    torch.manual_seed(1)
    model = A.Aligner(len(sym)).to(DEV)
    batch = corpus.batch(list(range(6)), DEV)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    loss, fs, bl, status = model.loss(*batch, bin_weight=1.0)
    loss.backward()
    assert A.status_bits(status) == 0
    with torch.no_grad():
        k, q = model.keys_queries(*A.Aligner._inputs(*batch))
        _, path = A.mas(A.AlignLogProbFn.apply(q, k, batch[1], batch[3], torch.zeros(7, dtype=torch.int32, device=DEV)), batch[1], batch[3],
                        torch.zeros(7, dtype=torch.int32, device=DEV))
    xs, il, mels, ol = (t.cpu() for t in batch)
    rt, rfs, rbl, params = O.loss(sd, xs, il, mels, ol, 1.0, path=path.cpu().numpy())
    rt.backward()
    e = abs(float(loss) - float(rt)) / abs(float(rt))
    _report("step_loss", e)
    assert e <= STEP_LOSS_GATE
    worst = 0.0
    for name, p in model.named_parameters():
        g = p.grad if name != "embed.weight" else p.grad[1:]
        r = params[name].grad if name != "embed.weight" else params[name].grad[1:]
        worst = max(worst, _rel(g, r))
    _report("step_grad", worst)
    assert worst <= STEP_GRAD_GATE
    opt = A.NoamAdam(model.parameters(), 256, 1.0, 10)
    losses = []
    for _ in range(4):
        loss, *_ = model.loss(*batch, bin_weight=1.0)
        losses.append(float(loss))
        opt.zero_grad()
        loss.backward()
        opt.clip_and_step(1.0)
    assert losses[3] < losses[0], losses


def test_recovers_durations_of_a_synthetic_corpus():
    lines = fixture_lines()
    sym = A.build_symbols(lines)
    corpus = A.Corpus(lines, sym, mels=render(lines, 0))
    model, hist = A.train(corpus, len(sym), steps=1000, batch=32, bin_start=500, seed=0, log=lambda m: None)
    durs = A.extract(model, corpus)
    agr = A.agreement(corpus.lines, durs)
    _report("recovery_within_1", agr["within_1"])
    print("MEASURED recovery", json.dumps(agr), hist[-1])
    assert 1 - agr["within_1"] <= MISS_GATE


def test_train_then_extract_on_a_tree(tmp_path, capsys):
    lines = fixture_lines(40)
    mels = render(lines, 1)
    (tmp_path / "mels").mkdir()
    for ln in lines:
        np.save(tmp_path / "mels" / f"{ln.id}.npy", mels[ln.id].T.copy())
    short = A.Line("", None, None, lines[0].phonemes * 20, "short.wav")     # more phonemes than frames
    np.save(tmp_path / "mels" / "short.npy", np.zeros((80, 10), np.float32))
    fl = tmp_path / "in.txt"
    fl.write_text("".join(A.format_line(ln, ln.durations) + "\n" for ln in lines) + A.format_line(short, [1] * len(short.phonemes)) + "\n")
    cfg = os.path.join(REPO, "fastspeech2_b200", "configs", "default.yaml")
    ck, out = tmp_path / "al.pt", tmp_path / "out.txt"
    A.main(["train", "-c", cfg, "--filelist", str(fl), "-d", str(tmp_path), "--steps", "20", "--batch", "8", "-o", str(ck)])
    A.main(["extract", "-c", cfg, "--filelist", str(fl), "-d", str(tmp_path), "-p", str(ck), "--out", str(out)])
    cap = capsys.readouterr()
    assert "skipping short.wav: " in cap.err
    agr = json.loads(cap.out.strip().splitlines()[-1])
    assert agr["lines"] == 40 and set(agr) >= {"within_1", "within_2", "mean_abs_boundary_frames", "worst_file"}
    got = A.read_filelist(str(out))
    assert [g.wav for g in got] == [ln.wav for ln in lines]
    for g in got:
        assert sum(g.durations) == mels[g.id].shape[0] and min(g.durations) >= 1
        assert g.boundaries == np.cumsum([0] + g.durations).tolist()
    model, symbols, step = A.load(str(ck))
    assert step == 20 and symbols == A.build_symbols(A.read_filelist(str(fl)))
