"""The fused optimizer step on the GPU (DESIGN.md §15, csrc/optim.cu, fastspeech2_b200/optim.py) against the reference's
own NoamOpt (core/optimizer.py, imported from the staged oracle/_ref) over torch's foreach Adam and clip_grad_norm_.
Bit-identical wherever the contract says so; the clipped path against torch is within a gate reported below.
Needs an H100: run with `-m gpu`."""
import copy
import importlib.util
import math
import os
import types

import numpy as np
import pytest
import torch

import _optim_plan as P
from fastspeech2_b200 import FeedForwardTransformer, _lib, synthetic_state_dict
from fastspeech2_b200 import optim as O
from fastspeech2_b200.hparams import load_hp
from fastspeech2_b200.sharded import GradientSync
from fastspeech2_b200.synthetic import make_batch

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_OPT = os.path.join(REPO, "oracle", "_ref", "core", "optimizer.py")
KEYS = ("xs", "ilens", "ys", "olens", "ds", "es", "ps")
D_MODEL, FACTOR, WARMUP = 384, 1.0, 4
CLIP_GATE = 4e-5          # 3x the worst observed (1.25e-5): |clipped NoamAdam - torch| over 20 steps, relative to max |update|


def ref_module():
    if not os.path.isfile(REF_OPT):
        pytest.skip("reference not staged in oracle/_ref")
    spec = importlib.util.spec_from_file_location("ref_core_optimizer", REF_OPT)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def holder(params):
    return types.SimpleNamespace(parameters=lambda: iter(params))


def model_params(seed=0):
    m = FeedForwardTransformer(68, 80, load_hp())
    m.load_state_dict(synthetic_state_dict(seed), strict=True)
    return [p.detach().to("cuda").clone().requires_grad_() for p in m.parameters()]


def twins(params):
    return [p.detach().clone().requires_grad_() for p in params]


def seeded_grads(params, step, scale=1e-3, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed * 1000 + step)
    return [torch.randn(p.shape, device="cuda", generator=g) * scale for p in params]


def set_grads(params, grads):
    for p, g in zip(params, grads):
        p.grad = g.clone()


def assert_same(ref, ours, ref_opt, our_opt, what=""):
    sd = our_opt.state_dict()["optimizer"]["state"]
    for i, (a, b) in enumerate(zip(ref, ours)):
        assert torch.equal(a, b) or (torch.isnan(a).any() and torch.equal(a.nan_to_num(), b.nan_to_num())), (what, i)
        sa = ref_opt.optimizer.state[a]
        if not sa:
            assert i not in sd
            continue
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(sa[k].nan_to_num(), sd[i][k].nan_to_num()), (what, i, k)
        assert sa["step"].dtype == sd[i]["step"].dtype == torch.float32 and sa["step"].device == sd[i]["step"].device
        assert float(sa["step"]) == float(sd[i]["step"]), (what, i)


# ---- 1. step() against NoamOpt.step() -------------------------------------------------------------------------------------------
def test_step_matches_reference_bit_for_bit():
    R = ref_module()
    ref = model_params()
    ours = twins(ref)
    ropt = R.get_std_opt(holder(ref), D_MODEL, WARMUP, FACTOR)
    oopt = O.get_std_opt(holder(ours), D_MODEL, WARMUP, FACTOR)
    for s in range(1, 21):
        grads = seeded_grads(ref, s)
        set_grads(ref, grads); set_grads(ours, grads)
        ropt.step(); oopt.step()
        assert oopt._step == ropt._step and oopt._rate == ropt._rate
        assert oopt.param_groups[0]["lr"] == ropt.param_groups[0]["lr"]
        assert_same(ref, ours, ropt, oopt, f"step {s}")
        ropt.zero_grad(); oopt.zero_grad()
        assert all(p.grad is None for p in ours)


@pytest.mark.parametrize("shape_off", [(1, 0), (3, 0), (1, 1), (3, 1), (7, 3), (P.CHUNK + 5, 1), (2 * P.CHUNK - 1, 2)])
def test_step_small_and_unaligned(shape_off):
    R = ref_module()
    n, off = shape_off
    base = torch.randn(n + 8, device="cuda")
    gbase = torch.empty(n + 8, device="cuda")
    ref = [base[off:off + n].clone().requires_grad_(), torch.randn(5, device="cuda").requires_grad_()]
    pb = base.clone()
    ours = [pb[off:off + n].requires_grad_(), ref[1].detach().clone().requires_grad_()]
    ropt = R.get_std_opt(holder(ref), D_MODEL, WARMUP, FACTOR)
    oopt = O.NoamAdam(ours, D_MODEL, FACTOR, WARMUP)
    for s in range(1, 8):
        grads = seeded_grads(ref, s, scale=1.0)
        set_grads(ref, grads)
        gbase[off:off + n].copy_(grads[0])
        ours[0].grad = gbase[off:off + n]
        ours[1].grad = grads[1].clone()
        ropt.step(); oopt.step()
        assert_same(ref, ours, ropt, oopt, f"n={n} off={off} step {s}")
    assert torch.equal(pb[:off], base[:off]) and torch.equal(pb[off + n:], base[off + n:])


# ---- per-step scalars -------------------------------------------------------------------------------------------------------
def test_device_scalars_steps_1_to_1e6():
    n = 10 ** 6
    for d, f, w in ((384, 1.0, 4000), (256, 1.0, 4), (384, 2.0, 4)):
        a, wp = P.noam_constants(d, f, w)
        hp = _lib.NoamAdamHp(a, wp, 0.9, 0.98, 1e-9)
        lr = torch.empty(n, dtype=torch.float64, device="cuda")
        ss, bc = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")
        _lib.check(_lib.load().fs2_optim_noam_scalars(1, n, hp, lr.data_ptr(), ss.data_ptr(), bc.data_ptr(), None), "scalars")
        steps = np.arange(1, n + 1)
        lr, ss, bc = lr.cpu().numpy(), ss.cpu().numpy(), bc.cpu().numpy()
        assert np.array_equal(lr, P.noam_rate(steps, d, f, w))
        py_lr = np.array([f * d ** (-0.5) * min(s ** (-0.5), s * w ** (-1.5)) for s in range(1, n + 1)])
        # Python's step ** -0.5 (libm pow) is not always correctly rounded: the double lr differs by one ulp at some steps,
        # the fp32 values torch consumes never do
        assert np.all(np.abs(lr - py_lr) <= 2 * np.spacing(py_lr))
        want_ss = np.array([(l / (1 - 0.9 ** float(s))) * -1 for s, l in zip(range(1, n + 1), py_lr)]).astype(np.float32)
        want_bc = np.array([(1 - 0.98 ** float(s)) ** 0.5 for s in range(1, n + 1)]).astype(np.float32)
        assert np.array_equal(ss, want_ss) and np.array_equal(bc, want_bc)


# ---- 2. norm ---------------------------------------------------------------------------------------------------------------------
def test_norm_is_within_one_ulp_and_deterministic():
    params = model_params()
    grads = seeded_grads(params, 1, scale=1.0)
    f64 = math.sqrt(sum(float((g.double() ** 2).sum()) for g in grads))
    norms = []
    side = torch.cuda.Stream()
    a = torch.randn(4096, 4096, device="cuda")
    for k in range(4):
        ps = twins(params)
        set_grads(ps, grads)
        opt = O.NoamAdam(ps, D_MODEL, FACTOR, WARMUP)
        if k % 2:                                  # other work in flight on another stream
            with torch.cuda.stream(side):
                for _ in range(4):
                    a = a @ a * 1e-3
        norms.append(opt.clip_and_step(1e9))
    torch.cuda.synchronize()
    bits = {int(n.view(torch.int32)) for n in norms}
    assert len(bits) == 1
    got = float(norms[0])
    ulp = float(np.spacing(np.float32(f64)))
    print(f"norm {got!r} float64 {f64!r} diff {abs(got - f64) / ulp:.3f} ulp")
    assert abs(got - f64) <= ulp


# ---- 3. clip_and_step against clip_grad_norm_ + NoamOpt.step() ---------------------------------------------------------------
def _torch_clip_loop(R, ref, ours, max_norm, steps=20):
    ropt = R.get_std_opt(holder(ref), D_MODEL, WARMUP, FACTOR)
    oopt = O.get_std_opt(holder(ours), D_MODEL, WARMUP, FACTOR)
    p0 = [p.detach().clone() for p in ref]
    worst = 0.0
    for s in range(1, steps + 1):
        grads = seeded_grads(ref, s, scale=1e-2)
        set_grads(ref, grads); set_grads(ours, grads)
        rn = torch.nn.utils.clip_grad_norm_(ref, max_norm)
        ropt.step()
        on = oopt.clip_and_step(max_norm)
        assert all(torch.equal(p.grad, g) for p, g in zip(ours, grads))      # .grad is not scaled in place
        upd = max(float((a.detach() - b).abs().max()) for a, b in zip(ref, p0))
        worst = max(worst, max(float((a.detach() - b.detach()).abs().max()) for a, b in zip(ref, ours)) / upd)
        assert float(rn) > 0 and abs(float(on) - float(rn)) <= 1e-5 * float(rn)
    return ropt, oopt, worst


def test_clip_above_norm_is_bit_identical():
    R = ref_module()
    ref = model_params()
    ours = twins(ref)
    ropt, oopt, worst = _torch_clip_loop(R, ref, ours, 1e6)
    assert worst == 0.0
    assert_same(ref, ours, ropt, oopt, "clip above the norm")


def test_clip_below_norm_within_gate():
    R = ref_module()
    ref = model_params()
    ours = twins(ref)
    _, _, worst = _torch_clip_loop(R, ref, ours, 0.5)
    print(f"clipped: worst |NoamAdam - torch| / max |update| = {worst:.3e} (gate {CLIP_GATE:.1e})")
    assert worst <= CLIP_GATE


# ---- 4. NaN guard and +inf ---------------------------------------------------------------------------------------------------------
def test_nan_gradient_skips_everything():
    R = ref_module()
    ref = model_params()
    ours = twins(ref)
    ropt = R.get_std_opt(holder(ref), D_MODEL, WARMUP, FACTOR)
    oopt = O.get_std_opt(holder(ours), D_MODEL, WARMUP, FACTOR)
    for s in range(1, 4):
        grads = seeded_grads(ref, s)
        if s == 2:
            grads[5].view(-1)[17] = float("nan")
        set_grads(ref, grads); set_grads(ours, grads)
        before = [p.detach().clone() for p in ours]
        sd_before = copy.deepcopy(oopt.state_dict())
        rn = torch.nn.utils.clip_grad_norm_(ref, 1.0)
        if not math.isnan(rn):                 # the reference loop's guard
            ropt.step()
        on = oopt.clip_and_step(1.0)
        if s == 2:
            assert math.isnan(float(on))
            assert all(torch.equal(a, b) for a, b in zip(before, ours))
            sd = oopt.state_dict()
            assert sd["_step"] == sd_before["_step"] == ropt._step
            for i, st in sd["optimizer"]["state"].items():
                for k in ("exp_avg", "exp_avg_sq", "step"):
                    assert torch.equal(st[k], sd_before["optimizer"]["state"][i][k])
        assert oopt._step == ropt._step and oopt.rate() == ropt.rate() and oopt._rate == ropt._rate


def test_inf_gradient_zero_coefficient_and_nan_parameter():
    R = ref_module()
    ref = model_params()
    ours = twins(ref)
    ropt = R.get_std_opt(holder(ref), D_MODEL, WARMUP, FACTOR)
    oopt = O.get_std_opt(holder(ours), D_MODEL, WARMUP, FACTOR)
    grads = seeded_grads(ref, 1)
    j = next(i for i, g in enumerate(grads) if g.numel() > 100)
    grads[j].view(-1)[9] = float("inf")
    set_grads(ref, grads); set_grads(ours, grads)
    rn = torch.nn.utils.clip_grad_norm_(ref, 1.0)
    ropt.step()
    on = oopt.clip_and_step(1.0)
    assert math.isinf(float(rn)) and math.isinf(float(on)) and oopt._step == 1
    assert math.isnan(float(ours[j].view(-1)[9]))
    assert_same(ref, ours, ropt, oopt, "inf")


def test_norm_above_fp32_range_torch_reports_inf():
    """torch sums the squares in fp32: a norm between ~1.8e19 and 3.4e38 overflows there; the fp64 sums stay finite."""
    p = [torch.zeros(4, device="cuda", requires_grad=True)]
    p[0].grad = torch.full((4,), 1e20, device="cuda")
    rn = torch.nn.utils.get_total_norm([p[0].grad])
    on = O.NoamAdam(p, D_MODEL, FACTOR, WARMUP).clip_and_step(1.0)
    print(f"norm of four 1e20: torch {float(rn)}, NoamAdam {float(on)}")
    assert math.isinf(float(rn)) and float(on) == pytest.approx(2e20, rel=1e-6)


# ---- 5. CUDA graph, no host sync --------------------------------------------------------------------------------------------------
def test_graph_replay_matches_eager_without_sync():
    params = model_params()
    eager, graphed = twins(params), twins(params)
    grads = [seeded_grads(params, s, scale=1e-2) for s in range(1, 5)]
    oe = O.NoamAdam(eager, D_MODEL, FACTOR, WARMUP)
    og = O.NoamAdam(graphed, D_MODEL, FACTOR, WARMUP)
    for p, g in zip(eager, grads[0]):
        p.grad = g.clone()
    static = [g.clone() for g in grads[0]]
    for p, g in zip(graphed, static):
        p.grad = g
    oe.clip_and_step(0.5)                      # warm-up: state, table, workspace
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        og.clip_and_step(0.5)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gnorm = og.clip_and_step(0.5)
    for s in range(1, 4):
        for p, g in zip(eager, grads[s]):
            p.grad.copy_(g)
        for t, g in zip(static, grads[s]):
            t.copy_(g)
        torch.cuda.set_sync_debug_mode("error")
        try:
            en = oe.clip_and_step(0.5)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(en, gnorm)
        assert all(torch.equal(a, b) for a, b in zip(eager, graphed)), s
    assert oe._step == og._step == 4


# ---- 6. checkpoints both ways ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("direction", ["reference_to_fused", "fused_to_reference"])
def test_checkpoint_round_trip(direction):
    R = ref_module()
    start = model_params()
    a, b = twins(start), twins(start)
    first = (R.get_std_opt(holder(a), D_MODEL, WARMUP, FACTOR) if direction == "reference_to_fused"
             else O.get_std_opt(holder(a), D_MODEL, WARMUP, FACTOR))
    for s in range(1, 4):
        set_grads(a, seeded_grads(a, s))
        first.step()
    sd = copy.deepcopy(first.state_dict())
    with torch.no_grad():
        for x, y in zip(b, a):
            x.copy_(y)
    second = (O.get_std_opt(holder(b), D_MODEL, WARMUP, FACTOR) if direction == "reference_to_fused"
              else R.get_std_opt(holder(b), D_MODEL, WARMUP, FACTOR))
    second.load_state_dict(sd)
    assert second._step == first._step == 3
    for s in range(4, 8):
        grads = seeded_grads(a, s)
        set_grads(a, grads); set_grads(b, grads)
        first.step(); second.step()
        assert all(torch.equal(x, y) for x, y in zip(a, b)), s
    fa, fb = first.state_dict(), second.state_dict()
    assert fa.keys() == fb.keys() and fa["_step"] == fb["_step"] and fa["_rate"] == fb["_rate"]
    assert fa["optimizer"]["param_groups"] == fb["optimizer"]["param_groups"]
    for i, st in fa["optimizer"]["state"].items():
        for k in ("exp_avg", "exp_avg_sq", "step"):
            assert torch.equal(st[k], fb["optimizer"]["state"][i][k]) and st[k].device == fb["optimizer"]["state"][i][k].device


# ---- 7. train steps -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bucket", [False, True])
def test_train_steps_match_torch_optimizer(bucket):
    """Three tf32 + flash train steps: the torch loop (clip_grad_norm_ + NoamOpt.step()) on one model, clip_and_step on its
    twin fed the same gradients (the backward runs once; its atomics make gradients of two separate runs differ in the
    last bits, which Adam's normalisation would amplify), as plain .grad tensors or as GradientSync bucket views."""
    from fastspeech2_b200 import train as T
    R = ref_module()
    batch = {k: v.to("cuda") for k, v in make_batch(4, 40, 200, seed=5).items()}

    def model():
        m = FeedForwardTransformer(68, 80, load_hp(), train_precision="tf32", train_attention="flash")
        m.load_state_dict(synthetic_state_dict(0), strict=True)
        return m.to("cuda").train()

    mt, mf = model(), model()
    sync = GradientSync(mf) if bucket else None
    ot, of = R.get_std_opt(mt, 384, 100, 1.0), O.get_std_opt(mf, 384, 100, 1.0)
    losses = []
    for s in range(3):
        mt.dropout_masks = T.MaskSource(seed=100)
        loss, _ = mt(*[batch[k] for k in KEYS])
        loss.backward()
        for a, b in zip(mt.parameters(), mf.parameters()):
            if a.grad is not None:
                if bucket:
                    b.grad.copy_(a.grad)
                else:
                    b.grad = a.grad.clone()
        torch.nn.utils.clip_grad_norm_(mt.parameters(), 1e30)
        ot.step()
        ot.zero_grad()
        of.clip_and_step(1e30)
        sync.zero_grad() if bucket else of.zero_grad()
        losses.append(float(loss.detach()))
        for (n, a), b in zip(mt.named_parameters(), mf.parameters()):
            assert torch.equal(a, b), (s, n)
    print("losses", losses)
    assert losses[-1] < losses[0]


# ---- 8. guard bands and .grad None -------------------------------------------------------------------------------------------------
def test_guard_bands_and_parameters_without_grad():
    G, S = 64, 12345.5
    sizes = [1, 3, 300, P.CHUNK + 7]
    bufs = {k: [torch.full((n + 2 * G,), S, device="cuda") for n in sizes] for k in ("p", "g", "m", "v")}
    params = []
    for j, n in enumerate(sizes):
        bufs["p"][j][G:G + n] = torch.randn(n, device="cuda")
        params.append(bufs["p"][j][G:G + n].requires_grad_())
    frozen = torch.randn(11, device="cuda", requires_grad=True)
    frozen0 = frozen.detach().clone()
    opt = O.NoamAdam(params + [frozen], D_MODEL, FACTOR, WARMUP)
    for s in range(1, 4):
        for j, n in enumerate(sizes):
            bufs["g"][j][G:G + n] = torch.randn(n, device="cuda")
            params[j].grad = bufs["g"][j][G:G + n]
        if s == 1:
            opt.clip_and_step(0.1)
            for j, (p, n) in enumerate(zip(params, sizes)):        # move the Adam state into guarded buffers
                st = opt.optimizer.state[p]
                for k, key in (("m", "exp_avg"), ("v", "exp_avg_sq")):
                    bufs[k][j][G:G + n] = st[key]
                    st[key] = bufs[k][j][G:G + n]
        else:
            opt.step() if s == 2 else opt.clip_and_step(0.1)
    torch.cuda.synchronize()
    for k in ("p", "g", "m", "v"):
        for j, n in enumerate(sizes):
            assert bool((bufs[k][j][:G] == S).all() and (bufs[k][j][G + n:] == S).all()), (k, j)
    assert torch.equal(frozen, frozen0) and frozen not in opt.optimizer.state


# ---- 9. the eval arena follows the update -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("entry", ["step", "clip_and_step"])
def test_eval_inference_sees_the_update(entry):
    m = FeedForwardTransformer(68, 80, load_hp())
    m.load_state_dict(synthetic_state_dict(0), strict=True)
    m = m.to("cuda").eval()
    x = make_batch(1, 20, 100, seed=9)["xs"][0].to("cuda")
    with torch.no_grad():
        before = m.inference(x)
    opt = O.get_std_opt(m, 384, 4, 1.0)
    for p, g in zip(m.parameters(), seeded_grads(list(m.parameters()), 1, scale=1e-2)):
        p.grad = g
    opt.step() if entry == "step" else opt.clip_and_step(1.0)
    with torch.no_grad():
        after = m.inference(x)
    fresh = FeedForwardTransformer(68, 80, load_hp())
    fresh.load_state_dict({k: v.cpu() for k, v in m.state_dict().items()}, strict=True)
    fresh = fresh.to("cuda").eval()
    with torch.no_grad():
        want = fresh.inference(x)
    assert not torch.equal(before, after) if before.shape == after.shape else True
    assert after.shape == want.shape and torch.equal(after, want)
