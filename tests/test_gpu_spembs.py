"""External speaker embeddings on the GPU (DESIGN.md section 27): parity with the unmodified reference (its encoder wrapped
to add the projected embeddings, tests/golden/spembs.npz), per-utterance bit-identity, the zero-projection identity with
the model without embeddings, the projection kernels against float64, the train step and its deterministic projection
gradients, graphed synthesis, and a training run that places two held-out embeddings.  Needs an H100: run with `-m gpu`."""
import ctypes as C
import json

import pytest
import torch

from fastspeech2_b200 import FeedForwardTransformer, _lib
from fastspeech2_b200 import optim as O
from fastspeech2_b200 import train as T
from fastspeech2_b200.hparams import load_hp
from fastspeech2_b200.synthetic import make_batch
from test_gpu_parity import PRECISIONS, TOL, close
from test_gpu_train_tc import ALPHA_GATE, GRAD_GATE, KBIAS_GATE, LOSS_GATE, REPORT_GATE
import _spembs_golden as EG

pytestmark = pytest.mark.gpu
T_ = torch.from_numpy
KEYS = ("xs", "ilens", "ys", "olens", "ds", "es", "ps")
U = 2.0 ** -24


def hp_with(d, n=0):
    hp = load_hp()
    hp["model"]["spk_embed_dim"] = d
    hp["model"]["n_speakers"] = n
    return hp


def make_model(weights, proj, table=None, prec="3xf16", **kw):
    """proj: (W, bias) or None (a model without spk_embed_dim)."""
    d = 0 if proj is None else int(proj[0].shape[1])
    m = FeedForwardTransformer(68, 80, hp_with(d, 0 if table is None else table.shape[0]), precision=prec, **kw)
    sd = dict(weights)
    if table is not None:
        sd["speaker_embed.weight"] = table
    if proj is not None:
        sd["spk_embed_proj.weight"], sd["spk_embed_proj.bias"] = proj
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


@pytest.fixture(scope="module")
def gold(golden):
    return golden("spembs")


@pytest.fixture(scope="module")
def models(weights):
    _, W, b = EG.seeded()
    return {(cfg, p): make_model(weights, (W, b), EG.table() if cfg == "both" else None, p) for cfg in EG.CONFIGS for p in PRECISIONS}


def batch(g, *keys):
    return [T_(g[k]).cuda() for k in keys]


def inputs(g, cfg):
    """The fixture's embeddings and, for the "both" configuration, its speaker ids."""
    e = EG.seeded()[0].cuda()
    spk = T_(g["speakers"]).cuda() if cfg == "both" else None
    return e, spk


def _mels(c, prefix, b, a, olens, prec):
    mels, means = EG.mel_checks(c, prefix, b, a, olens)
    for what, got, want in mels:
        close(got, want, TOL[prec], what)
    for what, got, want in means:
        close(got, want, dict(max=TOL[prec]["mean"], mean=TOL[prec]["mean"]), what)


# ---- 1. parity with the reference ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", PRECISIONS)
@pytest.mark.parametrize("cfg", EG.CONFIGS)
def test_golden_teacher_forced(models, gold, cfg, prec):
    c = EG.cfg(gold, cfg)
    xs, il, ol, ds, es, ps = batch(gold, "xs", "ilens", "olens", "ds", "es", "ps")
    e, spk = inputs(gold, cfg)
    with torch.no_grad():
        b, a, d, eo, po = models[cfg, prec]._forward(xs, il, ol, ds, es, ps, is_inference=False, speakers=spk, spembs=e)
    close(d, c["tf_d_outs"], TOL["fp32"], "d_outs")
    close(eo, c["tf_e_outs"], dict(max=2e-4, mean=2e-5), "e_outs")
    close(po, c["tf_p_outs"], dict(max=2e-4, mean=2e-5), "p_outs")
    _mels(c, "tf", b, a, ol, prec)


@pytest.mark.parametrize("prec", PRECISIONS)
@pytest.mark.parametrize("cfg", EG.CONFIGS)
def test_golden_inference(models, gold, cfg, prec):
    c = EG.cfg(gold, cfg)
    xs, il = batch(gold, "xs", "ilens")
    e, spk = inputs(gold, cfg)
    with torch.no_grad():
        b, a, d, eh, ph = models[cfg, prec]._forward(xs, il, is_inference=True, speakers=spk, spembs=e)
    assert torch.equal(d.cpu(), T_(c["inf_d_outs"])) and a.shape[1] == int(c["inf_frames"])
    _mels(c, "inf", b, a, d.sum(1), prec)


# ---- 2. per-utterance bit-identity ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", PRECISIONS)
@pytest.mark.parametrize("controlled", [False, True])
def test_synthesize_is_per_utterance(models, gold, prec, controlled):
    m = models["both", prec]
    xs, il = batch(gold, "xs", "ilens")
    e, spk = inputs(gold, "both")
    B = xs.shape[0]
    ctl = {}
    if controlled:
        speed = 0.8 + 0.5 * torch.rand(xs.shape, generator=torch.Generator().manual_seed(4)).cuda()
        speed[torch.arange(xs.shape[1], device="cuda")[None, :] >= il[:, None]] = float("nan")
        ctl = dict(speed=speed, pitch=1.1, energy=torch.linspace(0.9, 1.2, B).cuda())
    for order in (torch.arange(B), torch.arange(B).flip(0)):
        o = order.cuda()
        with torch.no_grad():
            mels, olens, dur = m.synthesize(xs[o], il[o], speakers=spk[o], spembs=e[o],
                                            **{k: (v[o] if torch.is_tensor(v) else v) for k, v in ctl.items()})
        for j, b in enumerate(order.tolist()):
            n = int(il[b])
            with torch.no_grad():
                kw = {k: (v[b, :n] if torch.is_tensor(v) and v.dim() == 2 else v[b] if torch.is_tensor(v) else v) for k, v in ctl.items()}
                alone = (m.inference_controlled(xs[b, :n], speaker=spk[b], spemb=e[b], **kw) if controlled
                         else m.inference(xs[b, :n], spk[b], e[b]))
            L = int(olens[j])
            assert L == alone.shape[0]
            assert torch.equal(mels[j, :L], alone), (prec, b)
            assert bool((mels[j, L:] == 0).all()) and not torch.signbit(mels[j, L:]).any()


# ---- 3. a zero projection is the model without embeddings --------------------------------------------------------------
@pytest.mark.parametrize("prec", PRECISIONS)
def test_zero_projection_equals_no_embeddings(weights, gold, prec):
    spe = make_model(weights, (torch.zeros(256, 192), torch.zeros(256)), prec=prec)
    plain = make_model(weights, None, prec=prec)
    xs, il, ol, ds, es, ps = batch(gold, "xs", "ilens", "olens", "ds", "es", "ps")
    e = EG.seeded()[0].cuda()
    with torch.no_grad():
        for got, want in ((spe.synthesize(xs, il, spembs=e), plain.synthesize(xs, il)),
                          ((spe.inference(xs[2, :int(il[2])], spemb=e[2]),), (plain.inference(xs[2, :int(il[2])]),)),
                          (spe._forward(xs, il, ol, ds, es, ps, spembs=e), plain._forward(xs, il, ol, ds, es, ps))):
            for a, b in zip(got, want):
                assert torch.equal(a, b), prec


def test_embeddings_change_the_mels(models, gold):
    xs, il = batch(gold, "xs", "ilens")
    e, _ = inputs(gold, "emb")
    n = int(il[0])
    with torch.no_grad():
        a, b = models["emb", "3xtf32"].inference(xs[0, :n], spemb=e[0]), models["emb", "3xtf32"].inference(xs[0, :n], spemb=e[2])
    L = min(a.shape[0], b.shape[0])
    assert float((a[:L] - b[:L]).abs().mean()) > 1e-2


def test_non_finite_embeddings_raise(models, gold):
    m = models["emb", "3xtf32"]
    xs, il, ol, ds, es, ps = batch(gold, "xs", "ilens", "olens", "ds", "es", "ps")
    e, _ = inputs(gold, "emb")
    for bad in (float("nan"), float("inf"), 3e19):        # 3e19 is finite, but its square overflows fp32
        e2 = e.clone()
        e2[4, 7] = bad
        with pytest.raises(ValueError, match="non-finite"), torch.no_grad():
            m.synthesize(xs, il, spembs=e2)
        with pytest.raises(ValueError, match="non-finite"), torch.no_grad():
            m._forward(xs, il, ol, ds, es, ps, spembs=e2)
        with pytest.raises(ValueError, match="non-finite"), torch.no_grad():
            m.inference(xs[4, :int(il[4])], spemb=e2[4])


# ---- 4. the kernels against float64 -------------------------------------------------------------------------------------
def _project(W, b, e):
    lib = _lib.load()
    B, D = e.shape
    v = torch.empty(B, W.shape[0], device="cuda")
    en = torch.empty(B, D, device="cuda")
    bad = torch.full((B,), 7, dtype=torch.int32, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    _lib.check(lib.fs2_spemb_project(W.data_ptr(), b.data_ptr(), e.data_ptr(), B, D, W.shape[0], v.data_ptr(), en.data_ptr(),
                                     bad.data_ptr(), status.data_ptr(), _lib.stream_ptr(e.device)), "fs2_spemb_project")
    return v, en, bad, status


@pytest.mark.parametrize("D", [1, 192, 512, 4096])
@pytest.mark.parametrize("B", [1, 7, 64])
def test_spemb_project_against_float64(D, B):
    g = torch.Generator().manual_seed(D * 100 + B)
    e = torch.randn(B, D, generator=g) * 4.0
    W, bias = torch.randn(256, D, generator=g), torch.randn(256, generator=g)
    if B > 1:
        e[1] = 0.0                                   # zero norm: normalize leaves it 0, v = bias
    if B > 2:
        e[B - 1, D // 2] = float("nan")
    v, en, bad, status = (t.cpu() for t in _project(W.cuda(), bias.cuda(), e.cuda()))
    nan_rows = torch.isnan(e).any(1)
    assert bad.tolist() == nan_rows.int().tolist()
    assert int(status[0]) == (_lib.FS2_SPEMB_NONFINITE if bool(nan_rows.any()) else 0)
    ok = ~nan_rows
    e64 = e[ok].double()
    en64 = e64 / e64.norm(dim=1, keepdim=True).clamp_min(1e-12)
    v64 = en64 @ W.double().T + bias.double()
    n = 2 * D + 8                                    # the norm's D terms, its sqrt and division, the D products
    bound_en = (D + 4) * U * en64.abs()
    assert bool(((en[ok].double() - en64).abs() <= bound_en + 1e-300).all())
    terms = en64.abs() @ W.double().abs().T + bias.double().abs()
    err = (v[ok].double() - v64).abs()
    assert bool((err <= n * U * terms).all()), float((err / (n * U * terms)).max())
    if B > 1:
        assert torch.equal(v[1], bias)
        for b in (0, B // 2):                        # each utterance's v depends on its embedding alone
            assert torch.equal(_project(W.cuda(), bias.cuda(), e[b:b + 1].cuda())[0].cpu()[0], v[b])


def test_spemb_project_flags_overflowing_norms():
    """A finite embedding whose fp32 sum of squares overflows would normalise to 0 and leave v = bias: it is flagged."""
    g = torch.Generator().manual_seed(9)
    e = torch.randn(5, 192, generator=g)
    e[1] = 1e20                      # every square overflows
    e[2, 3] = 3e19                   # one square overflows
    e[3, 3] = 1e19                   # 1e38 still fits: not flagged
    W, bias = torch.randn(256, 192, generator=g).cuda(), torch.randn(256, generator=g).cuda()
    v, en, bad, status = _project(W, bias, e.cuda())
    assert bad.tolist() == [0, 1, 1, 0, 0] and int(status[0]) == _lib.FS2_SPEMB_NONFINITE
    assert torch.isfinite(v[[0, 3, 4]]).all()


@pytest.mark.parametrize("D, B", [(1, 1), (192, 8), (512, 64), (4096, 16)])
def test_spemb_project_backward_against_float64(D, B):
    g = torch.Generator().manual_seed(D + B)
    dv, en = torch.randn(B, 256, generator=g), torch.randn(B, D, generator=g)
    lib = _lib.load()
    outs = []
    for _ in range(2):
        dW, db = torch.full((256, D), 0.5, device="cuda"), torch.full((256,), -0.25, device="cuda")
        dvc, enc = dv.cuda(), en.cuda()
        _lib.check(lib.fs2_spemb_project_backward(dvc.data_ptr(), enc.data_ptr(), B, D, 256, dW.data_ptr(), db.data_ptr(),
                                                  _lib.stream_ptr(dvc.device)), "fs2_spemb_project_backward")
        outs.append((dW.cpu(), db.cpu()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    dW64 = 0.5 + dv.double().T @ en.double()
    db64 = -0.25 + dv.double().sum(0)
    tW = 0.5 + dv.double().abs().T @ en.double().abs()
    tb = 0.25 + dv.double().abs().sum(0)
    assert bool(((outs[0][0].double() - dW64).abs() <= (B + 1) * U * tW).all())
    assert bool(((outs[0][1].double() - db64).abs() <= (B + 1) * U * tb).all())


def test_row_norm_spemb_adds_after_the_table():
    g = torch.Generator().manual_seed(3)
    B, L, Cc = 3, 5, 256
    x, gamma, beta = (torch.randn(B * L, Cc, generator=g).cuda(), torch.randn(Cc, generator=g).cuda(), torch.randn(Cc, generator=g).cuda())
    table, vec = torch.randn(4, Cc, generator=g).cuda(), torch.randn(B, Cc, generator=g).cuda()
    spk = torch.tensor([2, 0, 3]).cuda()
    lib = _lib.load()

    def run(spk_vec):
        out = torch.empty(B * L, Cc, device="cuda")
        d = _lib.RowNormDesc(x=x.data_ptr(), ldx=Cc, gamma=gamma.data_ptr(), beta=beta.data_ptr(), eps=1e-5, rows=B * L, C=Cc,
                             out=out.data_ptr(), ldo=Cc, spk_table=table.data_ptr(), spk=spk.data_ptr(), n_spk=4, spk_L=L)
        _lib.check(lib.fs2_op_row_norm_spemb(C.byref(d), spk_vec, _lib.stream_ptr(x.device)), "fs2_op_row_norm_spemb")
        return out

    plain = torch.empty(B * L, Cc, device="cuda")
    d = _lib.RowNormDesc(x=x.data_ptr(), ldx=Cc, gamma=gamma.data_ptr(), beta=beta.data_ptr(), eps=1e-5, rows=B * L, C=Cc,
                         out=plain.data_ptr(), ldo=Cc, spk_table=table.data_ptr(), spk=spk.data_ptr(), n_spk=4, spk_L=L)
    _lib.check(lib.fs2_op_row_norm(C.byref(d), _lib.stream_ptr(x.device)), "fs2_op_row_norm")
    assert torch.equal(run(None), plain)
    want = plain + vec.repeat_interleave(L, 0)          # one fp32 add after the table's
    assert torch.equal(run(vec.data_ptr()), want)


def test_workspace_holds_the_projected_vectors(weights):
    spe = make_model(weights, (torch.zeros(256, 192), torch.zeros(256)))
    plain = make_model(weights, None)
    lib, x = _lib.load(), torch.zeros(1, 1, dtype=torch.int64, device="cuda")
    for B, Tn in ((1, 1), (64, 100), (300, 7)):
        got = []
        for m in (spe, plain):
            n = C.c_size_t()
            _lib.check(lib.fs2_workspace_bytes(m._ready(x), B, Tn, 0, C.byref(n)), "fs2_workspace_bytes")
            got.append(n.value)
        assert B * 256 * 4 <= got[0] - got[1] <= B * 256 * 4 + 255, (B, Tn, got)


def test_encode_refuses_mismatched_embeddings(models, gold):
    m = models["emb", "3xtf32"]
    xs, il = batch(gold, "xs", "ilens")
    h, lib = m._ready(xs), _lib.load()
    ws = m._ws(8, xs.shape[1], 0)
    hs = torch.empty(8, xs.shape[1], 256, device="cuda")
    e = EG.seeded()[0].cuda()
    for ptr, d, words in ((None, 192, "pass spembs"), (e.data_ptr(), 191, "D=191 but the loaded projection takes D=192")):
        rc = lib.fs2_encode_spemb(h, xs.data_ptr(), il.data_ptr(), None, ptr, d, 8, xs.shape[1], hs.data_ptr(), None, None,
                                  ws.data_ptr(), ws.numel(), 0, None, None, _lib.stream_ptr(xs.device))
        assert rc == -1 and words in lib.fs2_last_error().decode()


# ---- 5. train step -------------------------------------------------------------------------------------------------------
class _Recorded(T.MaskSource):
    def __init__(self, masks):
        super().__init__(seed=0, injected=None)
        self.recorded = list(masks)

    def next(self, shape, p, device):
        self.calls += 1
        m = self.recorded.pop(0)
        if tuple(m.shape) != tuple(shape):
            m = m.permute(0, 2, 1)
        return m.to(torch.uint8).contiguous().to(device)

    def attention(self, shape, p, device):
        return self.next(shape, p, device), 0, 0


def _golden_step(weights, g, train_precision, train_attention=None):
    gen = torch.Generator().manual_seed(5)
    recorded = [torch.rand(shape, generator=gen) >= p for shape, p in zip(json.loads(str(g["mask_shapes"])), g["mask_rates"].tolist())]
    e, W, bias = EG.seeded()
    m = FeedForwardTransformer(68, 80, hp_with(EG.D, 5), precision="fp32", train_precision=train_precision,
                               train_attention=train_attention)
    sd = dict(weights)
    sd["speaker_embed.weight"] = EG.table()
    sd["spk_embed_proj.weight"], sd["spk_embed_proj.bias"] = W, bias
    m.load_state_dict(sd, strict=True)
    m = m.cuda().train()
    m.dropout_masks = _Recorded(recorded)
    bt = EG.batch(g)
    args = [bt[k].cuda() for k in KEYS]
    ys, ol = args[2], args[3]
    ys[torch.arange(ys.shape[1], device="cuda")[None, :] >= ol[:, None]] = float("nan")
    loss, rep = m(*args, speakers=T_(g["speakers"]).cuda(), spembs=e.cuda())
    loss.backward()
    torch.cuda.synchronize()
    assert not m.dropout_masks.recorded
    return m, loss, rep


def _errors(m, g):
    no_grad = set(json.loads(str(g["no_grad"])))
    samples = EG.grad_samples(g, {n: p.numel() for n, p in m.named_parameters()})
    full = {k: T_(g["grad/" + k]).reshape(-1) for k in ("speaker_embed.weight", "spk_embed_proj.bias")}
    errs, kbias = {}, 0.0
    for name, p in m.named_parameters():
        if name in no_grad:
            assert p.grad is None, name
            continue
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
        flat = p.grad.detach().reshape(-1).cpu()
        if name in full:
            scale = float(full[name].abs().max())
            err = float((flat - full[name]).abs().max())
        else:
            idx, vals, scale = samples[name]
            err = max(float((flat[idx] - vals).abs().max()), abs(float(flat.abs().max()) - scale))
        if name.endswith("self_attn.linear_k.bias"):
            kbias = max(kbias, err / samples[name.replace(".bias", ".weight")][2])
            continue
        errs[name] = (err, scale)
    return errs, kbias


def test_train_step_fp32_matches_reference(weights, gold):
    m, loss, rep = _golden_step(weights, gold, "fp32")
    assert abs(float(loss) - float(gold["loss"])) <= 1e-4 * abs(float(gold["loss"]))
    for a, vb in zip(rep, gold["report_values"].tolist()):
        assert abs(list(a.values())[0] - vb) <= 1e-4 * max(1.0, abs(vb))
    errs, _ = _errors(m, gold)
    for name, (err, scale) in errs.items():
        gate = 3e-2 if name.startswith("postnet.") else 1e-2      # test_gpu_speakers.py's gates
        assert err <= gate * scale + 1e-6, (name, err, scale)
    print("projection gradient errors (fp32):", errs["spk_embed_proj.weight"], errs["spk_embed_proj.bias"])


@pytest.mark.parametrize("attention", ["materialized", "flash"])
def test_train_step_tf32_matches_reference(weights, gold, attention):
    m, loss, rep = _golden_step(weights, gold, "tf32", attention)
    lerr = abs(float(loss) - float(gold["loss"])) / abs(float(gold["loss"]))
    rerr = max(abs(list(a.values())[0] - vb) / max(1.0, abs(vb)) for a, vb in zip(rep, gold["report_values"].tolist()))
    errs, kbias = _errors(m, gold)
    rel = {n: e / (s + 1e-12) for n, (e, s) in errs.items()}
    alpha = max(rel.pop(n) for n in list(rel) if n.endswith(".alpha"))
    worst = max(rel.items(), key=lambda kv: kv[1])
    print(f"tf32 {attention}: loss rel {lerr:.2e}, report rel {rerr:.2e}, worst {worst}, proj W {rel['spk_embed_proj.weight']:.2e}, "
          f"proj b {rel['spk_embed_proj.bias']:.2e}, alpha {alpha:.2e}, key bias {kbias:.2e}")
    assert lerr <= LOSS_GATE and rerr <= REPORT_GATE
    assert worst[1] <= GRAD_GATE and alpha <= ALPHA_GATE and kbias <= (KBIAS_GATE if attention == "materialized" else 1e-3)


@pytest.mark.parametrize("B, Tn, D", [(1, 1, 1), (8, 37, 192), (64, 200, 512), (16, 131, 4096)])
def test_spemb_add_fn_against_float64(B, Tn, D):
    """The forward is one fp32 add of v; the projection's gradients against float64 autograd through normalize and the
    linear map, gated at n 2^-24 sum|terms| with n = T + B + D + 8 (the sum over T, the sum over b and the normalisation)."""
    g = torch.Generator().manual_seed(B * Tn + D)
    x, dy = torch.randn(B, Tn, 256, generator=g), torch.randn(B, Tn, 256, generator=g)
    e, W, bias = torch.randn(B, D, generator=g) * 2, torch.randn(256, D, generator=g), torch.randn(256, generator=g)
    Wr, br = W.double().requires_grad_(), bias.double().requires_grad_()
    en64 = torch.nn.functional.normalize(e.double())
    (x.double() + (en64 @ Wr.T + br).unsqueeze(1)).backward(dy.double())
    Wc, bc = W.cuda().requires_grad_(), bias.cuda().requires_grad_()
    v, en, status = T.spemb_project(Wc, bc, e.cuda())
    assert int(status[0]) == 0
    got = T.SpembAddFn.apply(x.cuda(), v, en, Wc, bc)
    assert torch.equal(got.cpu(), (x.cuda() + v.unsqueeze(1)).cpu())
    got.backward(dy.cuda())
    n = Tn + B + D + 8
    tW = dy.double().abs().sum(1).T @ en64.abs()
    tb = dy.double().abs().sum((0, 1))
    assert bool(((Wc.grad.cpu().double() - Wr.grad).abs() <= n * U * tW + 1e-30).all())
    assert bool(((bc.grad.cpu().double() - br.grad).abs() <= n * U * tb + 1e-30).all())


def _three_steps(weights, e):
    torch.manual_seed(11)
    _, W, bias = EG.seeded()
    m = FeedForwardTransformer(68, 80, hp_with(EG.D, 5), precision="fp32", train_precision="tf32", train_attention="flash",
                               train_deterministic=True)
    sd = dict(weights)
    sd["speaker_embed.weight"] = EG.table()
    sd["spk_embed_proj.weight"], sd["spk_embed_proj.bias"] = W, bias
    m.load_state_dict(sd, strict=True)
    m = m.cuda().train()
    m.dropout_masks = T.MaskSource(seed=3)
    opt = O.NoamAdam(m.parameters(), 384, 1.0, 100)
    losses = []
    for step in range(3):
        bt = make_batch(8, 19, 120, seed=50 + step)
        loss, _ = m(*[bt[k].cuda() for k in KEYS], speakers=torch.tensor([0, 3, 3, 1, 0, 2, 3, 1]).cuda(), spembs=e)
        opt.zero_grad()
        loss.backward()
        opt.clip_and_step(1.0)
        losses.append(float(loss))
    return losses, {k: v.detach().clone() for k, v in m.state_dict().items()}


def test_two_deterministic_runs_give_equal_bits(weights):
    e = EG.seeded()[0].cuda()
    a, b = _three_steps(weights, e), _three_steps(weights, e)
    assert a[0] == b[0]
    assert all(torch.equal(a[1][k], b[1][k]) for k in a[1])
    assert not torch.equal(a[1]["spk_embed_proj.weight"], EG.seeded()[1].cuda())


def test_train_step_refuses_non_finite_embeddings(weights):
    m = make_model(weights, EG.seeded()[1:]).train()
    bt = make_batch(2, 10, 40, seed=2)
    e = EG.seeded()[0][:2].cuda()
    e[1, 0] = float("nan")
    with pytest.raises(ValueError, match="non-finite"):
        m(*[bt[k].cuda() for k in KEYS], spembs=e)


# ---- 6. graphed synthesis ------------------------------------------------------------------------------------------------
def test_graphed_synthesis_with_embeddings(models, gold):
    m = models["both", "3xtf32"]
    xs, il = batch(gold, "xs", "ilens")
    e, spk = inputs(gold, "both")
    B, Tn = xs.shape
    gs = m.graphed_synthesize(B, Tn, 400)
    graph = gs.graph
    mels, olens, dur = (t.clone() for t in gs(xs, il, spk, spembs=e))
    for b in range(B):
        n, L = int(il[b]), int(olens[b])
        with torch.no_grad():
            alone, ol1, _ = m.synthesize(xs[b:b + 1, :n], il[b:b + 1], speakers=spk[b:b + 1], spembs=e[b:b + 1])
        assert L == int(ol1[0]) and torch.equal(mels[b, :L], alone[0, :L]), b
        assert bool((mels[b, L:] == 0).all())
    other = e.flip(0).contiguous()
    mels2, olens2, _ = (t.clone() for t in gs(xs, il, spk, spembs=other))
    assert gs.graph is graph and not torch.equal(mels2, mels)
    with torch.no_grad():
        alone, ol1, _ = m.synthesize(xs[:1, :int(il[0])], il[:1], speakers=spk[:1], spembs=other[:1])
    assert torch.equal(mels2[0, :int(ol1[0])], alone[0, :int(ol1[0])])
    bad = e.clone()
    bad[3, 11] = float("nan")
    with pytest.raises(ValueError, match="non-finite"):
        gs(xs, il, spk, spembs=bad)
    assert bool((gs.mels[3] == 0).all()) and int(gs.olens[3]) == 0
    keep = [b for b in range(B) if b != 3]
    assert torch.equal(gs.mels[keep], mels[keep]) and torch.equal(gs.olens[keep], olens[keep])
    gs(xs, il, spk, validate=False, spembs=bad)                 # no check at all
    il0 = il.clone()
    il0[3] = 0                                                  # an empty slot needs no finite embedding
    gs(xs, il0, spk, spembs=bad)
    with pytest.raises(ValueError, match="pass them"):
        gs(xs, il, spk)


# ---- 7. zero-shot: held-out embeddings ----------------------------------------------------------------------------------
# 32 training speakers with D = 4 normalised embeddings: many more than the D + 1 = 5 coefficients of an affine map, so the
# training data fix the offset of every other embedding.  Targets: N(0, 0.09) mels plus 2 u_hat . e_hat.
ZS_D, ZS_SPEAKERS, ZS_STEPS, ZS_WARMUP, ZS_FACTOR = 4, 32, 300, 200, 0.15
ZS_U = torch.tensor([1.0, -0.8, 0.6, 0.3])
ZS_GATE = 0.5
ZS_COS = (0.45, -0.45)                     # the held-out embeddings' cosines with u: targets +0.9 and -0.9


def _zs_embeddings():
    """ZS_SPEAKERS training embeddings and two held-out ones, each normalised, and their offsets 2 u_hat . e_hat."""
    g = torch.Generator().manual_seed(21)
    unit = ZS_U / ZS_U.norm()
    train = torch.nn.functional.normalize(torch.randn(ZS_SPEAKERS, ZS_D, generator=g))
    held = []
    for c in ZS_COS:
        w = torch.randn(ZS_D, generator=g)
        w = torch.nn.functional.normalize(w - (w @ unit) * unit, dim=0)
        held.append(c * unit + (1 - c * c) ** 0.5 * w)
    held = torch.stack(held)
    return train, held, 2.0 * train @ unit, 2.0 * held @ unit


def zero_shot_means(weights, steps=ZS_STEPS, factor=ZS_FACTOR, warmup=ZS_WARMUP, proj_std=1.0):
    """Train deterministically (TF32, NoamAdam + clip_and_step) from the synthetic weights and an N(0, proj_std^2)
    projection; -> (teacher-forced mel means of the held-out embeddings, their targets, the training targets)."""
    train, held, t_off, h_off = _zs_embeddings()
    m = FeedForwardTransformer(68, 80, hp_with(ZS_D), precision="3xf16", train_precision="tf32", train_deterministic=True)
    sd = dict(weights)
    g = torch.Generator().manual_seed(5)
    sd["spk_embed_proj.weight"] = torch.randn(256, ZS_D, generator=g) * proj_std
    sd["spk_embed_proj.bias"] = torch.zeros(256)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().train()
    m.dropout_masks = T.MaskSource(seed=3)
    opt = O.NoamAdam(m.parameters(), 384, factor, warmup)
    for step in range(steps):
        bt = make_batch(8, 24, 120, seed=100 + step)
        s = torch.randint(0, ZS_SPEAKERS, (8,), generator=g)
        bt["ys"] = torch.randn(bt["ys"].shape, generator=g) * 0.3 + t_off[s][:, None, None]
        bt["es"].zero_(); bt["ps"].zero_()
        loss, _ = m(*[bt[k].cuda() for k in KEYS], spembs=train[s].cuda())
        opt.zero_grad()
        loss.backward()
        opt.clip_and_step(1.0)
    m.eval()
    bt = make_batch(4, 24, 120, seed=7)
    bt["es"].zero_(); bt["ps"].zero_()
    means = []
    with torch.no_grad():
        for k in range(len(held)):
            _, after, *_ = m._forward(*[bt[k2].cuda() for k2 in ("xs", "ilens", "olens", "ds", "es", "ps")],
                                      spembs=held[k].expand(4, ZS_D).contiguous().cuda())
            means.append(float(after.mean()))
    return means, h_off.tolist(), t_off.tolist()


def test_zero_shot_offsets_from_held_out_embeddings(weights):
    means, targets, _ = zero_shot_means(weights)
    print("held-out mel means:", [f"{v:.3f}" for v in means], "targets", [f"{v:.3f}" for v in targets])
    # calibration (H100 80GB HBM3, 700 W, DESIGN.md section 27): the run is deterministic and gave means 0.991 and -0.698
    # for targets +0.9 and -0.9 (errors 0.09 and 0.20, gap 1.69 for 1.8).  Gates: each mean within 0.5 of its linear
    # target, and the gap at least half the targets' gap
    assert max(abs(a - b) for a, b in zip(means, targets)) <= ZS_GATE, means
    assert means[0] - means[1] >= 0.5 * (targets[0] - targets[1]), means
