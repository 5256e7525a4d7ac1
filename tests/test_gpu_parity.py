"""Parity of the CUDA path (through the C ABI) against the golden vectors of the reference
and against the CPU oracle on seeded inputs.  Needs an H100: run with `-m gpu`.

Tolerances (stated, per SURVEY.md section 7 "fp32 tolerance vs tensor cores"):
  FS2_MATH_FP32 : max-abs <= 1e-4 on mels (output rms ~0.6; the oracle's own fp32 noise floor
                  vs fp64 is 2.4e-6, long K=3456 fp32 reductions in a different order add ~1e-5)
  FS2_MATH_3XTF32 ("3xf16", the default): max-abs <= 1e-4, mean-abs <= 1e-5 -- the reference-precision gate: every
                  contraction incl. attention error-compensated; what remains is the tensor core's fp32 accumulation
  FS2_MATH_TF32 : max-abs <= 1e-2, mean-abs <= 1e-3 on mels (tf32 operands: 10-bit mantissa, truncation)
  FS2_MATH_F16  : max-abs <= 5e-3, mean-abs <= 5e-4 (decoder side on fp16 hi planes: 10-bit mantissa, round-to-nearest)
  integer outputs (durations, bucket ids, LengthRegulator rows): bit-exact in every mode.
"""
import numpy as np
import pytest
import torch

from fastspeech2_b200 import FeedForwardTransformer, LengthRegulator, _lib
from fastspeech2_b200.hparams import load_hp
from fastspeech2_b200.synthetic import make_batch
from oracle import fs2_oracle as O

pytestmark = pytest.mark.gpu
T_ = torch.from_numpy
TOL = {"fp32": dict(max=1e-4, mean=1e-5), "tf32": dict(max=1e-2, mean=1e-3), "3xtf32": dict(max=1e-4, mean=1e-5),
       "f16": dict(max=5e-3, mean=5e-4)}
PRECISIONS = ["fp32", "tf32", "3xtf32", "f16"]
LOSS_REL = {"fp32": 1e-4, "tf32": 2e-3, "3xtf32": 1e-4, "f16": 2e-3}     # relative tolerance on the seven loss terms


def close(got, want, tol, what=""):
    got = got.detach().float().cpu().numpy().astype(np.float64)
    want = np.asarray(want.detach().cpu().numpy() if torch.is_tensor(want) else want, dtype=np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    err = np.abs(got - want)
    assert err.max() <= tol["max"] and err.mean() <= tol["mean"], f"{what}: max {err.max():.3e} mean {err.mean():.3e}"


@pytest.fixture(scope="module")
def models(weights):
    out = {}
    for prec in PRECISIONS:
        m = FeedForwardTransformer(68, 80, load_hp(), precision=prec)
        m.load_state_dict(weights, strict=True)
        out[prec] = m.cuda().eval()
    return out


def cuda(d, *keys):
    return [T_(d[k]).cuda() if isinstance(d[k], np.ndarray) else d[k].cuda() for k in keys]


# ---- golden vectors of the unmodified reference -------------------------------------------------
@pytest.mark.parametrize("prec", PRECISIONS)
def test_golden_teacher_forced(models, golden, prec):
    g = golden("tf_ragged")
    xs, il, ol, ds, es, ps = cuda(g, "xs", "ilens", "olens", "ds", "es", "ps")
    with torch.no_grad():
        b, a, d, e, p = models[prec]._forward(xs, il, ol, ds, es, ps, is_inference=False)
    close(d, g["d_outs"], TOL["fp32"], "d_outs")       # encoder + predictors: fp32 or 3xTF32 in every mode
    close(e, g["e_outs"], dict(max=2e-4, mean=2e-5), "e_outs")
    close(p, g["p_outs"], dict(max=2e-4, mean=2e-5), "p_outs")
    close(b, g["before"], TOL[prec], "before")
    close(a, g["after"], TOL[prec], "after")


@pytest.mark.parametrize("prec", PRECISIONS)
def test_golden_filelist_twin(models, golden, prec):
    """SURVEY 8d ragged twin of c2: first 64 rows of the reference's train filelist (real phonemes and durations,
    T 31..116, L 222..856) through the live reference; the fixture keeps all d_outs, two mels, eight e/p rows and
    per-utterance means of everything else (tests/golden/make_golden.py::filelist_twin)."""
    from _synth import seeded_energy_pitch
    g = golden("filelist64")
    olens = T_(g["olens"])
    L = int(olens.max())
    es, ps = seeded_energy_pitch(int(g["es_seed"]), olens, L)
    xs, il, ol, ds = cuda(g, "xs", "ilens", "olens", "ds")
    with torch.no_grad():
        b, a, d, e, p = models[prec]._forward(xs, il, ol, ds, es.cuda(), ps.cuda(), is_inference=False)
    close(d, g["d_outs"], TOL["fp32"], "d_outs")
    rows = T_(g["ep_rows"]).cuda()
    close(e[rows], g["e_sel"], dict(max=2e-4, mean=2e-5), "e_outs")
    close(p[rows], g["p_sel"], dict(max=2e-4, mean=2e-5), "p_outs")
    lo, hi = (int(v) for v in g["mel_rows"])
    close(a[lo, :olens[lo]], g["after_lo"], TOL[prec], "after[shortest]")
    close(a[hi, :olens[hi]], g["after_hi"], TOL[prec], "after[longest]")
    close(b[lo, :olens[lo]], g["before_lo"], TOL[prec], "before[shortest]")
    valid = (torch.arange(L)[None, :] < olens[:, None]).double().cuda()
    n = olens.double().cuda()
    mean_tol = dict(max=TOL[prec]["mean"], mean=TOL[prec]["mean"])          # a mean over >= 222*80 values
    close((a.double() * valid[..., None]).sum((1, 2)) / (n * 80), g["after_mean"], mean_tol, "after means")
    close((a.double().abs() * valid[..., None]).sum((1, 2)) / (n * 80), g["after_absmean"], mean_tol, "after abs means")
    close((b.double() * valid[..., None]).sum((1, 2)) / (n * 80), g["before_mean"], mean_tol, "before means")
    close((e.double() * valid).sum(1) / n, g["e_mean"], dict(max=2e-5, mean=2e-5), "e means")
    close((p.double() * valid).sum(1) / n, g["p_mean"], dict(max=2e-5, mean=2e-5), "p means")


@pytest.mark.parametrize("prec", PRECISIONS)
def test_golden_inference_ragged(models, golden, prec):
    g = golden("inf_ragged")
    xs, il = cuda(g, "xs", "ilens")
    with torch.no_grad():
        b, a, d, eh, ph = models[prec]._forward(xs, il, is_inference=True)
    assert d.dtype == torch.int64 and torch.equal(d.cpu(), T_(g["d_outs"]))          # bit-exact durations
    assert eh.shape == (3, g["before"].shape[1], 256) and eh.dtype == torch.float32
    assert torch.equal(eh.argmax(-1).cpu(), T_(g["e_ids"])) and torch.equal(ph.argmax(-1).cpu(), T_(g["p_ids"]))
    assert float(eh.sum()) == eh.shape[0] * eh.shape[1]
    close(b, g["before"], TOL[prec], "before")
    close(a, g["after"], TOL[prec], "after")


@pytest.mark.parametrize("prec", PRECISIONS)
def test_golden_inference_single(models, golden, prec):
    g = golden("inf_single")
    with torch.no_grad():
        mel = models[prec].inference(T_(g["x"]).cuda())
    close(mel, g["mel"], TOL[prec], "mel")


@pytest.mark.parametrize("prec", PRECISIONS)
def test_golden_forward_loss(models, golden, prec):
    g, gl = golden("tf_ragged"), golden("tf_ragged_loss")
    xs, il, ys, ol, ds, es, ps = cuda(g, "xs", "ilens", "ys", "olens", "ds", "es", "ps")
    with torch.no_grad():
        loss, report = models[prec](xs, il, ys, ol, ds, es, ps)
    import json, os
    from conftest import GOLDEN
    assert [list(r.keys())[0] for r in report] == json.load(open(os.path.join(GOLDEN, "report_keys.json")))
    rel = LOSS_REL[prec]
    got = np.array([list(r.values())[0] for r in report])
    assert np.all(np.abs(got - gl["report"]) <= rel * np.maximum(1.0, np.abs(gl["report"]))), (got, gl["report"])
    assert abs(float(loss) - float(gl["loss"])) <= rel * max(1.0, abs(float(gl["loss"])))
    assert loss.dim() == 0 and loss.is_cuda


@pytest.mark.parametrize("prec", PRECISIONS)
def test_reference_unit_test_twin(models, golden, prec):
    """tests/test_fastspeech2.py:7-20 with the same shapes/dtypes (float durations!) on CUDA, eval, no_grad."""
    gl = golden("unit_shapes")
    x = torch.ones(2, 100, dtype=torch.int64).cuda(); il = torch.tensor([100, 100]).cuda()
    y = torch.ones(2, 100, 80).cuda(); dur = torch.ones(2, 100).cuda(); e = torch.ones(2, 100).cuda(); p = torch.ones(2, 100).cuda()
    with torch.no_grad():
        loss, report = models[prec](x, il, y, il.clone(), dur, e, p)
    rel = LOSS_REL[prec]
    got = np.array([list(r.values())[0] for r in report])
    assert np.all(np.abs(got - gl["report"]) <= rel * np.maximum(1.0, np.abs(gl["report"]))), (got, gl["report"])


def test_golden_length_regulator_bit_exact(golden):
    g = golden("length_regulator")
    lr = LengthRegulator()
    hs, il = T_(g["hs"]).cuda(), T_(g["ilens"]).cuda()
    d = T_(g["d_int"]).cuda()
    assert torch.equal(lr(hs, d, il).cpu(), T_(g["out_int"]))
    assert torch.equal(d.cpu(), T_(g["d_int_after"]))             # in-place all-zero -> ones
    d = T_(g["d_int"]).cuda()
    assert torch.equal(lr(hs, d, il, alpha=2.5).cpu(), T_(g["out_alpha"]))
    assert torch.equal(d.cpu(), T_(g["d_alpha_after"]))           # alpha != 1: caller's ds untouched
    d = T_(g["d_float"]).cuda()
    assert torch.equal(lr(hs, d, il).cpu(), T_(g["out_float"]))
    assert torch.equal(d.cpu(), T_(g["d_float_after"]))
    with pytest.raises(RuntimeError, match="negative"):
        lr(hs, torch.full((4, 9), -1, dtype=torch.int64).cuda(), il)


def test_golden_bucketize(models, golden):
    g = golden("bucketize")
    m = models["fp32"]
    assert torch.equal(m.energy_predictor.to_one_hot(T_(g["vals_e"]).cuda()).argmax(-1).cpu(), T_(g["ids_e"]))
    assert torch.equal(m.pitch_predictor.to_one_hot(T_(g["vals_p"]).cuda()).argmax(-1).cpu(), T_(g["ids_p"]))


# ---- CPU oracle on seeded inputs ------------------------------------------------------------------
def test_length_regulator_c5_stress_bit_exact():
    """BASELINE config 5: B=256, T=100, ds~U{1..15}, alpha=4 (round half even) -> Lmax ~3.7k; ragged twin with
    zeros and an all-zero row.  Full size, bit-exact against the oracle, plus the mutated ds."""
    g = torch.Generator().manual_seed(5)
    hs = torch.randn(256, 100, 256, generator=g)
    lr = LengthRegulator()
    for ragged in (False, True):
        ds = torch.randint(1, 16, (256, 100), generator=g)
        il = torch.full((256,), 100, dtype=torch.int64)
        if ragged:
            il = torch.randint(30, 101, (256,), generator=g); il[0] = 100
            ds[torch.rand(256, 100, generator=g) < 0.1] = 0
            ds[7, :] = 0
        want_ds = ds.clone()
        want = O.length_regulator(hs, want_ds, il, alpha=4.0)
        got_ds = ds.clone().cuda()
        got = lr(hs.cuda(), got_ds, il.cuda(), alpha=4.0)
        assert got.shape == want.shape and torch.equal(got.cpu(), want)
        assert torch.equal(got_ds.cpu(), want_ds)
        want_ds = ds.clone(); want = O.length_regulator(hs, want_ds, il)       # alpha == 1 path mutates
        got_ds = ds.clone().cuda(); got = lr(hs.cuda(), got_ds, il.cuda())
        assert torch.equal(got.cpu(), want) and torch.equal(got_ds.cpu(), want_ds)


@pytest.mark.parametrize("prec", PRECISIONS)
def test_oracle_teacher_forced_ragged_batch(models, weights, prec):
    """B=8 ragged LJSpeech-like batch (padding leaks into valid frames in the reference; the rectangle
    must be reproduced): every output against the oracle on the identical padded batch."""
    ilens = [60, 57, 49, 41, 33, 25, 12, 5]
    olens = [480, 470, 401, 300, 259, 211, 90, 37]
    bt = make_batch(8, 60, 480, seed=21, ilens=ilens, olens=olens)
    torch.set_num_threads(8)
    with torch.no_grad():
        want = O.forward_path(weights, bt["xs"], bt["ilens"], bt["olens"], bt["ds"].clone(), bt["es"], bt["ps"], False)
        got = models[prec]._forward(bt["xs"].cuda(), bt["ilens"].cuda(), bt["olens"].cuda(), bt["ds"].cuda(), bt["es"].cuda(),
                                    bt["ps"].cuda(), is_inference=False)
    close(got[2], want[2], TOL["fp32"], "d_outs")
    close(got[3], want[3], dict(max=2e-4, mean=2e-5), "e_outs"); close(got[4], want[4], dict(max=2e-4, mean=2e-5), "p_outs")
    close(got[0], want[0], TOL[prec], "before"); close(got[1], want[1], TOL[prec], "after")


@pytest.mark.parametrize("prec", PRECISIONS)
def test_oracle_long_form(models, weights, prec):
    """config-4 shape at reduced batch: L = 2000 frames (attention tiles, positional table, Postnet)."""
    bt = make_batch(2, 250, 2000, seed=22, ilens=[250, 190], olens=[2000, 1603])
    with torch.no_grad():
        want = O.forward_path(weights, bt["xs"], bt["ilens"], bt["olens"], bt["ds"].clone(), bt["es"], bt["ps"], False)
        got = models[prec]._forward(*[bt[k].cuda() for k in ("xs", "ilens", "olens", "ds", "es", "ps")], is_inference=False)
    close(got[0], want[0], TOL[prec], "before"); close(got[1], want[1], TOL[prec], "after")


def test_repack_after_weight_update(models, weights):
    m = models["fp32"]
    bt = make_batch(2, 20, 150, seed=23)
    args = [bt[k].cuda() for k in ("xs", "ilens", "olens", "ds", "es", "ps")]
    with torch.no_grad():
        a0 = m._forward(*args)[1].clone()
        m.feat_out.bias.add_(1.0)                      # in-place update bumps the version counter
        a1 = m._forward(*args)[1].clone()
        m.feat_out.bias.sub_(1.0)
        a2 = m._forward(*args)[1]
    assert float((a1 - a0).abs().min()) > 0.5 and torch.allclose(a2, a0, atol=1e-6)


# ---- single kernels against plain PyTorch fp32 ----------------------------------------------------
def _tap_gemm(mode, x, w, bias, act, resid):
    lib = _lib.load()
    B, L, K = x.shape
    taps, N, _ = w.shape
    out = torch.empty(B, L, N, device="cuda")
    _lib.check(lib.fs2_op_tap_gemm(mode, _lib.ptr(x), B, L, K, _lib.ptr(w), _lib.ptr(bias), N, taps, act, _lib.ptr(resid),
                                   _lib.ptr(out), _lib.stream_ptr(x.device)), "fs2_op_tap_gemm")
    return out


@pytest.mark.parametrize("prec", ["fp32", "tf32"])
@pytest.mark.parametrize("shape", [(3, 70, 256, 1024, 9, 1), (2, 333, 384, 384, 1, 0), (5, 41, 80, 256, 5, 2),
                                   (2, 130, 256, 80, 5, 0), (1, 7, 1024, 384, 1, 0), (4, 100, 256, 256, 3, 1)])
def test_tap_gemm_vs_torch(prec, shape):
    B, L, K, N, taps, act = shape
    g = torch.Generator().manual_seed(hash(shape) & 0xffff)
    x = torch.randn(B, L, K, generator=g); w = torch.randn(N, K, taps, generator=g) / (K * taps) ** 0.5
    bias = torch.randn(N, generator=g); resid = torch.randn(B, L, N, generator=g)
    y = torch.nn.functional.conv1d(x.transpose(1, 2).double(), w.double(), bias.double(), padding=(taps - 1) // 2).transpose(1, 2)
    y = torch.relu(y) if act == 1 else torch.tanh(y) if act == 2 else y
    y = (y + resid.double()).float()
    wp = w.permute(2, 0, 1).contiguous().cuda()
    got = _tap_gemm(_lib.MATH_MODES[prec], x.cuda(), wp, bias.cuda(), act, resid.cuda())
    tol = dict(max=2e-5, mean=2e-6) if prec == "fp32" else dict(max=1e-2, mean=1e-3)
    close(got, y, tol, str(shape))


@pytest.mark.parametrize("shape", [(3, 70, 256, 1024, 9, 1), (2, 333, 256, 768, 1, 0), (5, 41, 256, 256, 3, 1),
                                   (1, 7, 1024, 256, 1, 0), (2, 130, 256, 80, 5, 0)])
def test_tap_gemm_3xtf32_is_fp32_class(shape):
    """The error-compensated tensor-core family used for the encoder / predictors in tf32 mode.  Operand
    rounding is compensated (hi/lo split), what remains is the tensor core's fp32 accumulation, which rounds
    toward zero: measured 2e-5 .. 2e-4 max-abs at K = 256 .. 2304 -- ~10x the CUDA-core FMA chain, ~50x tighter
    than plain tf32.  Stated tolerance: max 5e-4, mean 5e-5."""
    B, L, K, N, taps, act = shape
    g = torch.Generator().manual_seed(hash(shape) & 0xffff)
    x = torch.randn(B, L, K, generator=g) * 2; w = torch.randn(N, K, taps, generator=g) / (K * taps) ** 0.5
    bias = torch.randn(N, generator=g); resid = torch.randn(B, L, N, generator=g)
    y = torch.nn.functional.conv1d(x.transpose(1, 2).double(), w.double(), bias.double(), padding=(taps - 1) // 2).transpose(1, 2)
    y = torch.relu(y) if act == 1 else y
    y = (y + resid.double()).float()
    wp = w.permute(2, 0, 1).contiguous().cuda()
    got3 = _tap_gemm(2, x.cuda(), wp, bias.cuda(), act, resid.cuda())
    got32 = _tap_gemm(0, x.cuda(), wp, bias.cuda(), act, resid.cuda())
    e3, e32 = float((got3.cpu() - y).abs().max()), float((got32.cpu() - y).abs().max())
    print(f"3xtf32 max err {e3:.3e} vs fp32-FMA {e32:.3e} for {shape}")
    close(got3, y, dict(max=5e-4, mean=5e-5), str(shape))


@pytest.mark.parametrize("shape", [(3, 70, 384, 1024, 9, 1), (2, 333, 1024, 384, 1, 0), (5, 41, 256, 256, 3, 1),
                                   (1, 128, 64, 128, 1, 0), (4, 300, 384, 1024, 9, 1), (1, 7, 1024, 384, 1, 0)])
def test_tap_gemm_f16_vs_torch(shape):
    """f16 family (decoder conv-FFN in FS2_MATH_F16): fp16 copies of x and w, fp32 accumulation.  Against
    float64 on the *same fp16-rounded operands* only the accumulation order / rounding remains (max 5e-4, mean 5e-5,
    as for 3xTF32), which pins descriptors, swizzle and the K stepping; against the unrounded operands the error is
    the 10-bit-mantissa class of the tf32 family (max 1e-2, mean 1e-3)."""
    B, L, K, N, taps, act = shape
    g = torch.Generator().manual_seed(hash(shape) & 0xffff)
    x = torch.randn(B, L, K, generator=g) * 2; w = torch.randn(N, K, taps, generator=g) / (K * taps) ** 0.5
    bias = torch.randn(N, generator=g); resid = torch.randn(B, L, N, generator=g)

    def ref(xx, ww):
        y = torch.nn.functional.conv1d(xx.transpose(1, 2).double(), ww.double(), bias.double(), padding=(taps - 1) // 2).transpose(1, 2)
        y = torch.relu(y) if act == 1 else y
        return (y + resid.double()).float()
    wp = w.permute(2, 0, 1).contiguous().cuda()
    got = _tap_gemm(_lib.MATH_MODES["f16"], x.cuda(), wp, bias.cuda(), act, resid.cuda())
    close(got, ref(x.half().float(), w.half().float()), dict(max=5e-4, mean=5e-5), f"{shape} vs fp16-rounded operands")
    close(got, ref(x, w), dict(max=1e-2, mean=1e-3), f"{shape} vs exact operands")


@pytest.mark.parametrize("prec", ["fp32", "tf32", "3xtf32", "f16"])
@pytest.mark.parametrize("C,L,masked", [(256, 100, True), (384, 333, True), (384, 800, False), (256, 37, False), (384, 129, True)])
def test_attention_vs_torch(prec, C, L, masked):
    B, H = 3, 2
    g = torch.Generator().manual_seed(C + L)
    qkv = torch.randn(B, L, 3 * C, generator=g)
    lens = torch.tensor([L, max(1, L // 2), max(1, L // 7)])
    q, k, v = [t.view(B, L, H, C // H).transpose(1, 2).double() for t in qkv.split(C, dim=-1)]
    s = q @ k.transpose(-1, -2) / (C // H) ** 0.5
    if masked:
        valid = torch.arange(L)[None] < lens[:, None]
        m = (valid[:, None, :] & valid[:, :, None])[:, None]
        p = torch.softmax(s.masked_fill(~m, -float("inf")), -1).masked_fill(~m, 0.0)
    else:
        p = torch.softmax(s, -1)
    want = (p @ v).transpose(1, 2).reshape(B, L, C).float()
    lib = _lib.load()
    ctx = torch.empty(B, L, C, device="cuda")
    qkv_c, lens_c = qkv.cuda(), lens.cuda()
    _lib.check(lib.fs2_op_attention(_lib.MATH_MODES[prec], _lib.ptr(qkv_c), _lib.ptr(lens_c) if masked else None, B, L, C, H,
                                    _lib.ptr(ctx), _lib.stream_ptr(ctx.device)), "fs2_op_attention")
    # 3xtf32 = error-compensated tensor-core attention (fp16 hi + lo planes for Q, K, V^T and P): fp32-class
    tol = {"fp32": dict(max=2e-5, mean=2e-6), "3xtf32": dict(max=5e-5, mean=5e-6)}.get(prec, dict(max=1e-2, mean=1e-3))
    close(ctx, want, tol, f"attention C={C} L={L} masked={masked}")


@pytest.mark.parametrize("prec,N", [("tf32", 384), ("f16", 384), ("3xtf32", 384), ("f16", 256), ("3xtf32", 256)])
@pytest.mark.parametrize("rows,K,with_resid", [(1000, 384, True), (51, 1024, True), (4097, 256, False), (40000, 384, True), (20000, 1024, True)])
def test_fused_gemm_layernorm_vs_torch(prec, N, rows, K, with_resid):
    """GEMM + residual + LayerNorm (out-projection / conv-FFN w_2) through fs2_op_gemm_layernorm: the tensor-core GEMM
    (tf32, f16, 3xF16) with the residual added in its epilogue, then the row LayerNorm kernel, which also writes the operand
    planes.  40000 rows = more tiles than SMs: every pipeline ring wraps several times; K = 1024 gives long K loops."""
    g = torch.Generator().manual_seed(rows + K + N)
    x = torch.randn(rows, K, generator=g); w = torch.randn(N, K, generator=g) / K ** 0.5; bias = torch.randn(N, generator=g)
    resid = torch.randn(rows, N, generator=g) + 2.0          # non-zero row mean: exercises the merge of the partial statistics
    gamma = 1 + 0.1 * torch.randn(N, generator=g); beta = torch.randn(N, generator=g)
    xc, wc, bc, rc, gc, btc = x.cuda(), w.cuda(), bias.cuda(), resid.cuda(), gamma.cuda(), beta.cuda()
    y = xc.double() @ wc.double().T + bc.double() + (rc.double() if with_resid else 0)
    want = torch.nn.functional.layer_norm(y, (N,), gc.double(), btc.double(), 1e-5).float()
    out = torch.full((rows, N), float("nan"), device="cuda")
    planes = torch.full((rows, N), float("nan"), device="cuda") if prec != "tf32" else None
    lib = _lib.load()
    _lib.check(lib.fs2_op_gemm_layernorm(_lib.MATH_MODES[prec], _lib.ptr(xc), rows, K, N, _lib.ptr(wc), _lib.ptr(bc), _lib.ptr(rc) if with_resid else None,
                                         _lib.ptr(gc), _lib.ptr(btc), 1e-5, _lib.ptr(out), _lib.ptr(planes) if planes is not None else None,
                                         _lib.stream_ptr(out.device)), "fs2_op_gemm_layernorm")
    tol = dict(max=3e-5, mean=3e-6) if prec == "3xtf32" else dict(max=1e-2, mean=1e-3)
    close(out, want, tol, f"gemm+ln {prec} N={N} rows={rows} K={K}")
    if planes is not None:      # the operand planes written for the next contraction carry the same rows (22 / 11 mantissa bits)
        rel = 2e-6 if prec == "3xtf32" else 1.5e-3
        assert torch.isfinite(planes).all()
        assert float(((planes - out).abs() - rel * out.abs()).max()) <= 1e-6, float((planes - out).abs().max())


# ---- edge cases -------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", PRECISIONS)
def test_edge_shapes_vs_oracle(models, weights, prec):
    """Smallest and most lopsided shapes: single phoneme, single frame rows, one long + one tiny utterance,
    lengths that are not multiples of any tile size."""
    cases = [
        dict(B=1, T=1, L=3, ilens=[1], olens=[3]),
        dict(B=2, T=3, L=5, ilens=[3, 1], olens=[5, 1]),
        dict(B=3, T=37, L=301, ilens=[37, 2, 19], olens=[301, 2, 130]),
        dict(B=1, T=129, L=1025, ilens=[129], olens=[1025]),
    ]
    for i, c in enumerate(cases):
        bt = make_batch(c["B"], c["T"], c["L"], seed=40 + i, ilens=c["ilens"], olens=c["olens"])
        with torch.no_grad():
            want = O.forward_path(weights, bt["xs"], bt["ilens"], bt["olens"], bt["ds"].clone(), bt["es"], bt["ps"], False)
            got = models[prec]._forward(*[bt[k].cuda() for k in ("xs", "ilens", "olens", "ds", "es", "ps")], is_inference=False)
        valid = (torch.arange(c["L"])[None] < bt["olens"][:, None])
        for name, g, w in (("before", got[0], want[0]), ("after", got[1], want[1])):
            close(g.cpu()[valid], w[valid], TOL[prec], f"case {i} {name}")
        close(got[2], want[2], TOL["fp32"], f"case {i} d_outs")


def test_inference_batch_matches_oracle_durations(models, weights):
    """is_inference=True on a ragged B=8 batch: integer durations must be identical to the CPU oracle in both
    precision modes (encoder + duration predictor run exact-fp32 / 3xTF32), mels within tolerance given equal L."""
    g = torch.Generator().manual_seed(77)
    ilens = [64, 50, 47, 33, 21, 12, 5, 1]
    xs = torch.zeros(8, 64, dtype=torch.int64)
    for b, n in enumerate(ilens):
        xs[b, :n] = torch.randint(1, 68, (n,), generator=g)
    il = torch.tensor(ilens)
    with torch.no_grad():
        want = O.forward_path(weights, xs, il, is_inference=True)
        for prec in PRECISIONS:
            got = models[prec]._forward(xs.cuda(), il.cuda(), is_inference=True)
            assert torch.equal(got[2].cpu(), want[2]), prec
            assert torch.equal(got[3].argmax(-1).cpu(), want[3].argmax(-1)) and torch.equal(got[4].argmax(-1).cpu(), want[4].argmax(-1)), prec
            close(got[1], want[1], TOL[prec], f"after {prec}")


def test_positional_table_extends_like_reference(weights):
    """core/embedding.py:48-66: an input longer than the stored sinusoid table regenerates it.  5100 frames > the 5000
    rows of the checkpoint; checked against the oracle (whose table is generated for the needed length too)."""
    m = FeedForwardTransformer(68, 80, load_hp(), precision="fp32")
    m.load_state_dict(weights, strict=True)
    m = m.cuda().eval()
    bt = make_batch(1, 10, 5100, seed=31)
    sd = dict(weights)
    from fastspeech2_b200.weights import positional_table
    sd["decoder.embed.4.pe"] = positional_table(5100, 384)
    with torch.no_grad():
        want = O.forward_path(sd, bt["xs"], bt["ilens"], bt["olens"], bt["ds"].clone(), bt["es"], bt["ps"], False)
        got = m._forward(*[bt[k].cuda() for k in ("xs", "ilens", "olens", "ds", "es", "ps")], is_inference=False)
    assert m.decoder.embed[-1].pe.shape[1] == 5100 and m.encoder.embed[-1].pe.shape[1] == 5000
    close(got[1], want[1], TOL["fp32"], "after, 5100 frames")


def test_sharded_synthesis_single_rank(models, weights):
    """synthesize_sharded with no process group == plain batched inference."""
    from fastspeech2_b200.sharded import synthesize_sharded
    g = torch.Generator().manual_seed(78)
    xs = torch.randint(1, 68, (4, 30), generator=g); il = torch.tensor([30, 30, 30, 30])
    mels, olens = synthesize_sharded(models["fp32"], xs.cuda(), il.cuda())
    with torch.no_grad():
        want = O.forward_path(weights, xs, il, is_inference=True)
    assert torch.equal(olens.cpu(), want[2].sum(1))
    close(mels, want[1], TOL["fp32"], "sharded mels")


@pytest.mark.parametrize("prec", PRECISIONS)
def test_cuda_graph_replay_matches_eager(models, prec):
    """One captured CUDA graph per shape: replay with new inputs must equal the eager path bit for bit, and the
    deferred length validation must still raise."""
    m = models[prec]
    a = make_batch(4, 30, 260, seed=91, ilens=[30, 22, 9, 30], olens=[260, 180, 77, 259])
    b = make_batch(4, 30, 260, seed=92, ilens=[30, 30, 30, 12], olens=[260, 260, 255, 101])
    A = [a[k].cuda() for k in ("xs", "ilens", "olens", "ds", "es", "ps")]
    B_ = [b[k].cuda() for k in ("xs", "ilens", "olens", "ds", "es", "ps")]
    g = m.graphed_forward(*A)
    with torch.no_grad():
        for inp in (B_, A, B_):
            want = [t.clone() for t in m._forward(*inp, is_inference=False)]
            got = g(*inp)
            for w, o in zip(want, got):
                assert torch.equal(w, o)
    bad = [t.clone() for t in A]
    bad[3][0, 0] += 5                                 # durations no longer sum to olens
    with pytest.raises(RuntimeError, match="length mismatch"):
        g(*bad)


def test_random_shapes_tf32_vs_fp32_paths(models):
    """Shape stress: 24 random (B, T, L) with ragged lengths through the kernel families (tf32 and f16 vs fp32) (the exact-fp32 CUDA-core
    path is already pinned to the oracle; the tensor-core path must agree with it within the tf32 tolerance).  Catches
    tile-boundary bugs: packed tail tiles, partial attention tiles, single-tile cases, odd L (transposed-V row pitch)."""
    g = torch.Generator().manual_seed(2024)
    for case in range(24):
        B = int(torch.randint(1, 7, (1,), generator=g))
        T = int(torch.randint(1, 90, (1,), generator=g))
        ilens = [T] + [int(torch.randint(1, T + 1, (1,), generator=g)) for _ in range(B - 1)]
        olens = [il * int(torch.randint(1, 12, (1,), generator=g)) + int(torch.randint(0, 5, (1,), generator=g)) for il in ilens]
        L = max(olens)
        olens[olens.index(L)] = L
        bt = make_batch(B, T, L, seed=500 + case, ilens=ilens, olens=olens)
        args = [bt[k].cuda() for k in ("xs", "ilens", "olens", "ds", "es", "ps")]
        with torch.no_grad():
            ref = models["fp32"]._forward(*args, is_inference=False)
            gots = {prec: models[prec]._forward(*args, is_inference=False) for prec in ("tf32", "f16")}
        valid = (torch.arange(L)[None] < bt["olens"][:, None]).cuda()
        for prec, got in gots.items():
            for name, r, o in (("before", ref[0], got[0]), ("after", ref[1], got[1])):
                err = (r - o).abs()[valid]
                assert torch.isfinite(o).all(), (case, prec, name)
                assert float(err.max()) <= 1e-2 and float(err.mean()) <= 1e-3, (case, prec, B, T, L, name, float(err.max()), float(err.mean()))
            assert float((ref[2] - got[2]).abs().max()) <= 2e-4, (case, prec, "d_outs")
