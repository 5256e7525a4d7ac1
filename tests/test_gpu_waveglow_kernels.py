"""WaveGlow's own stages (csrc/waveglow.cu) against float64, one flow at a time, through fs2_op_waveglow_flow and
fs2_op_waveglow_upsample, which run fs2_waveglow's code for that stage on a handle loaded by fs2_waveglow_load (so the
production packing is under test too: cond bias + in bias, the skip rows [C, 2C) of res_skip, wg_pack_up_kernel):

  * the entries are the vocoder: upsampling, then flows 11 .. 0 from fp32(z), reproduce fs2_waveglow's audio bit for bit;
  * wg_flow_kernel alone (end conv, affine coupling, inverse 1x1 conv) for c = 8, 6, 4 at every channel count of the
    coverage table, against float64 on the same fp32 inputs, bit-identical across the four modes, in place and out of
    place, columns < 8 - c untouched, +0 past lens, NaN past lens inert;
  * a whole flow (start, the 8 WN layers with their cond / in-layer / res / skip GEMMs and gates, the flow kernel) at C in
    {64, 192, 256, 320, 512, 1024} (res / skip tiles 64, 80 and 128 wide), flows 11, 7 and 3, all four modes: the WN skip
    sum and the new state, on lens in steps shorter than the dilations 2 .. 128, with Ls not a multiple of 128, and one
    case of more than 2 x 132 row tiles;
  * the upsampling at olens below the 4 taps, its planes bit for bit against a restatement of split_pair;
  * per-utterance bits (alone, in the batch, in the reversed batch), sentinel guard bands around every output, bad
    lengths and the range bit of the status word.

The float64 references run on the GPU with the oracle's modules (oracle/waveglow_oracle.py: WN[k], convinv[k].infer,
upsample with the trim and grouping of `infer`) on the fp32 tensors the library loads.  Gates are relative to a float64
bound on the size of each element: the error over the summed |terms| of the operation that produced it (the skip GEMMs
for the skip sum; end, the coupling by |audio_1 - b| / exp(s) and |y| |s|, and |W^-1| for the state; the upsampling
GEMM for cond), against the exact operands and, in f16 / tf32,
against the operands those modes multiply (fp16 hi planes at scale 16 with each weight at its power-of-two scale;
tf32-truncated fp32).  Gate values are at most 3x the errors measured on an H100 (DESIGN.md section 9).

Weights: as tests/test_gpu_waveglow.py draws them (every weight-normed conv at torch's default init with g moved off |v|
by U[0.5, 1.5), `end` N(0, 1 / C) with bias N(0, 0.1^2)), drawn on the GPU so that C = 1024 costs seconds."""
import math
import zlib

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from fastspeech2_b200 import _lib
from fastspeech2_b200.waveglow import HOP, N_FLOWS, N_LAYERS, STEPS, flow_channels
from oracle import waveglow_oracle as O
from test_gpu_tap_gemm import MODE, TF32_CONVERSION, Guarded, bits, f16_operands, split_planes, to_tf32

DEV = "cuda"
MODES = ("fp32", "tf32", "f16", "3xf16")
RANGE, BAD_LENGTH = _lib.FS2_WAVEGLOW_RANGE, _lib.FS2_WAVEGLOW_BAD_LENGTH
COND = 640
PER_FLOW = 2 + 6 * N_LAYERS + 3                    # fs2_waveglow_load's tensors per flow

# ---- case tables (tests/test_waveglow_args.py checks what they cover) ----------------------------------------------
LS = 300                                           # step rows per utterance: not a multiple of 128
# lens in steps: 0; one in [2^(i-1), 2^i) for every dilation 2^i, i = 1 .. 7; a full 128-row tile and one row either
# side; two rows short of and one row past two tiles; the whole buffer
LENS = (300, 0, 1, 3, 6, 12, 31, 40, 127, 128, 129, 255, 257)
WN_CS = (64, 192, 256, 320, 512, 1024)             # res / skip tiles (N = C) 64, 64, 128, 80, 128, 128 wide
TAIL_CS = (64, 192, 256, 320, 448, 512, 960, 1024) # wg_flow_kernel alone (no GEMM), up to its largest shared memory
FLOWS = (11, 7, 3)                                 # c = 4, 6, 8
BIG = (3, 12000)                                   # (B, Ls): 94 row tiles per utterance (93 full, a 96-row tail)
BIG_LENS = (12000, 11873, 11001)                   # 94 + 93 + 86 = 273 live row tiles of the 282 the walk visits
UP_OLENS = (37, 1, 2, 3, 4, 5, 0)                  # frames; 1 .. 3 are fewer than the 4 taps the upsampling reads
UP_L = 37

# (max, mean) of the error over the magnitude bound per stage, mode and reference: 3x the largest value measured over
# the cases on an H100 80GB HBM3 (700 W), rounded down.  Over a whole flow the operands a mode multiplies explain only
# part of its error (2x less than exact in f16, 6x in tf32; one GEMM of the upsampling: all of it): every layer's
# operands are rounded from values that already differ from the reference's in their last fp32 bits
GATES = {
    "tail": {"exact": (2.9e-7, 2.2e-8)},
    "wn": {"fp32": {"exact": (3.2e-7, 4.9e-8)}, "3xf16": {"exact": (3.3e-6, 4.5e-7)},
           "f16": {"fp16 operands": (1.8e-4, 2.1e-5), "exact": (3.7e-4, 6.3e-5)},
           "tf32": {"tf32 operands": (2.1e-4, 2.3e-5), "exact": (1.3e-3, 2.1e-4)}},
    "state": {"fp32": {"exact": (3.6e-7, 6.5e-8)}, "3xf16": {"exact": (3.6e-6, 8.7e-7)},
              "f16": {"fp16 operands": (1.6e-4, 2.1e-5), "exact": (3.6e-4, 6.4e-5)},
              "tf32": {"tf32 operands": (1.6e-4, 2.4e-5), "exact": (1.2e-3, 2.3e-4)}},
    "upsample": {"fp32": {"exact": (7.6e-7, 4.6e-8)}, "3xf16": {"exact": (1.4e-6, 1.6e-7)},
                 "f16": {"fp16 operands": (7.3e-7, 5.9e-8), "exact": (5.2e-4, 5.4e-5)},
                 "tf32": {"tf32 operands": (9.8e-7, 1.1e-7), "exact": (1.3e-3, 1.4e-4)}},
}


# ---- weights and handles -------------------------------------------------------------------------------------------
def weights(C, seed):
    """fs2_waveglow_load's 638 device fp32 tensors (weight norm folded, torch layouts, W^-1 in float64 rounded once),
    drawn as test_gpu_waveglow.make_oracle draws them: a weight-normed conv folds to v * U[0.5, 1.5) per output channel
    with v and the bias U(+-1/sqrt(fan_in)); `end` N(0, 1/C), bias N(0, 0.1^2); convinv a QR rotation of det +1."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    uni = lambda shape, bound: (torch.rand(shape, generator=gen, device=DEV) * 2 - 1) * bound

    def conv(cout, cin, k):
        bound = 1 / math.sqrt(cin * k)
        w = uni((cout, cin, k), bound) * (torch.rand(cout, 1, 1, generator=gen, device=DEV) + 0.5)
        return [w.contiguous(), uni((cout,), bound).contiguous()]

    ts = [uni((80, 80, 1024), 1 / math.sqrt(80 * 1024)).contiguous(), uni((80,), 1 / math.sqrt(80 * 1024)).contiguous()]
    for k in range(N_FLOWS):
        c = flow_channels(k)
        ts += conv(C, c // 2, 1)
        for i in range(N_LAYERS):
            ts += conv(2 * C, C, 3)
        for i in range(N_LAYERS):
            ts += conv(2 * C, COND, 1)
        for i in range(N_LAYERS):
            ts += conv(2 * C if i < N_LAYERS - 1 else C, C, 1)
        ts += [(torch.randn(c, C, 1, generator=gen, device=DEV) / C ** 0.5).contiguous(),
               (torch.randn(c, generator=gen, device=DEV) * 0.1).contiguous()]
        W = torch.linalg.qr(torch.randn(c, c, generator=gen, device=DEV, dtype=torch.float64))[0]
        if torch.det(W) < 0:
            W[:, 0] = -W[:, 0]
        ts.append(torch.linalg.inv(W).float().contiguous())
    assert len(ts) == 2 + N_FLOWS * PER_FLOW
    return ts


class Net:
    """An fs2_waveglow_net created and loaded with tensors ts in one math mode."""

    def __init__(self, C, mode, ts):
        import ctypes as Ct
        lib = _lib.load()
        h = Ct.c_void_p()
        _lib.check(lib.fs2_waveglow_create(Ct.byref(h), MODE[mode], C), "fs2_waveglow_create")
        self.h, self.C, self.mode = h.value, C, mode
        tp = (Ct.c_void_p * len(ts))(*[t.data_ptr() for t in ts])
        _lib.check(lib.fs2_waveglow_load(self.h, tp, len(ts), _lib.stream_ptr(torch.device(DEV))), "fs2_waveglow_load")
        torch.cuda.synchronize()

    def __del__(self):
        _lib.load().fs2_waveglow_destroy(self.h)


_CACHE = {}


def model(C, seed=0):
    """(tensors, {mode: Net}) for one C at a time: the previous C's weights and handles are released first."""
    key = (C, seed)
    if key not in _CACHE:
        _CACHE.clear()
        torch.cuda.empty_cache()
        _CACHE[key] = (weights(C, 1000 * C + seed), {})
    return _CACHE[key]


def net(C, mode, seed=0):
    ts, nets = model(C, seed)
    if mode not in nets:
        nets[mode] = Net(C, mode, ts)
    return nets[mode]


@pytest.fixture(scope="module", autouse=True)
def _release():
    yield
    _CACHE.clear()
    torch.cuda.empty_cache()


# ---- the entries ---------------------------------------------------------------------------------------------------
def run_flow(n, k, cond, state_in, lens, *, skip_in=None, out=None, wn=True):
    """fs2_op_waveglow_flow on guarded outputs.  out: None (a sentinel-filled state_out: out of place), "inplace" (a
    guarded copy of state_in as both), or a Guarded to write into.  Returns (state_out [B, Ls, 8], wn [B, Ls, C] or
    None, status)."""
    lib = _lib.load()
    B, Ls, _ = state_in.shape
    if out == "inplace":
        g_st = Guarded(B * Ls * 8, torch.float32)
        g_st.view.copy_(state_in.reshape(-1))
        src = g_st.view
    else:
        g_st = out if out is not None else Guarded(B * Ls * 8, torch.float32)
        src = state_in
    g_wn = Guarded(B * Ls * n.C, torch.float32) if wn and skip_in is None else None
    status = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    before = lib.fs2_kernel_launches()
    _lib.check(lib.fs2_op_waveglow_flow(n.h, k, _lib.ptr(cond), _lib.ptr(skip_in), _lib.ptr(src), _lib.ptr(g_st.view), _lib.ptr(lens),
                                        B, Ls, _lib.ptr(g_wn.view) if g_wn else None, _lib.ptr(status), _lib.stream_ptr(state_in.device)),
               "fs2_op_waveglow_flow")
    launches = lib.fs2_kernel_launches() - before
    torch.cuda.synchronize()
    # prep + the flow kernel; with the WN: (cond planes,) start, 8 x (cond, in-layer, gate, skip), 7 res
    planes = n.mode in ("f16", "3xf16")
    assert launches == (2 if skip_in is not None else 2 + planes + 1 + 8 * 4 + 7)
    assert g_st.intact(), "a store landed outside state_out"
    assert g_wn is None or g_wn.intact(), "a store landed outside wn_out"
    return g_st.view.view(B, Ls, 8), (g_wn.view.view(B, Ls, n.C) if g_wn else None), int(status.item())


def run_upsample(n, mels, olens, planes=None):
    lib = _lib.load()
    B, L, _ = mels.shape
    planes = n.mode in ("f16", "3xf16") if planes is None else planes
    g = Guarded(B * L * STEPS * COND, torch.float32)
    gp = Guarded(B * L * STEPS * COND, torch.float32) if planes else None
    status = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    _lib.check(lib.fs2_op_waveglow_upsample(n.h, _lib.ptr(mels), _lib.ptr(olens), B, L, _lib.ptr(g.view), _lib.ptr(gp.view) if gp else None,
                                            _lib.ptr(status), _lib.stream_ptr(mels.device)), "fs2_op_waveglow_upsample")
    torch.cuda.synchronize()
    assert g.intact() and (gp is None or gp.intact()), "a store landed outside cond / cond_planes"
    return g.view.view(B, L * STEPS, COND), (gp.view.view(B, L * STEPS, COND) if gp else None), int(status.item())


# ---- float64 references --------------------------------------------------------------------------------------------
def q16(v):
    """an activation's hi plane back in fp32: rn_fp16(16 v) / 16"""
    return (v.float() * 16).clamp(-65504, 65504).half().float() / 16


def q16w(w):
    """a weight at its power-of-two scale, rounded to fp16 (the hi weight plane)"""
    return f16_operands(w[:1].flatten().float(), w.float())[1]


def tf32(v):
    return to_tf32(v.float().contiguous(), TF32_CONVERSION)


def operands(label):
    """(activation rounding, weight rounding) of a reference"""
    return {"exact": (lambda v: v, lambda w: w), "fp16 operands": (q16, q16w), "tf32 operands": (tf32, tf32)}[label]


def flow_tensors(ts, k):
    base = 2 + k * PER_FLOW
    t = ts[base: base + PER_FLOW]
    return {"start": t[0:2], "in": [t[2 + 2 * i: 4 + 2 * i] for i in range(N_LAYERS)],
            "cond": [t[18 + 2 * i: 20 + 2 * i] for i in range(N_LAYERS)], "rs": [t[34 + 2 * i: 36 + 2 * i] for i in range(N_LAYERS)],
            "end": t[50:52], "winv": t[52]}


def oracle_flow(ts, k, C, qa, qw):
    """(WN[k], convinv[k]) of the oracle in float64 on the GPU with the library's fp32 tensors, every GEMM's weight
    rounded by qw (res_skip's res rows [0, C) and skip rows [C, 2C) separately, as they are loaded) and every GEMM's
    input by qa (forward pre-hooks).  start and end run on CUDA cores in fp32 in every mode: not rounded.  convinv's
    weight is inv(W^-1) in float64, so that its `infer` multiplies by the library's W^-1."""
    f = flow_tensors(ts, k)
    c = flow_channels(k)
    with torch.device(DEV):
        wn = O.WN(c // 2, COND, N_LAYERS, C, 3)
        inv = O.Invertible1x1Conv(c)
    for m in [wn.start, *wn.in_layers, *wn.cond_layers, *wn.res_skip_layers]:
        nn.utils.remove_weight_norm(m)
    wn, inv = wn.double().eval(), inv.double().eval()
    with torch.no_grad():
        wn.start.weight.copy_(f["start"][0]); wn.start.bias.copy_(f["start"][1])
        for i in range(N_LAYERS):
            wn.in_layers[i].weight.copy_(qw(f["in"][i][0])); wn.in_layers[i].bias.copy_(f["in"][i][1])
            wn.cond_layers[i].weight.copy_(qw(f["cond"][i][0])); wn.cond_layers[i].bias.copy_(f["cond"][i][1])
            w = f["rs"][i][0]
            wn.res_skip_layers[i].weight.copy_(torch.cat([qw(w[:C]), qw(w[C:])]) if i < N_LAYERS - 1 else qw(w))
            wn.res_skip_layers[i].bias.copy_(f["rs"][i][1])
        wn.end.weight.copy_(f["end"][0]); wn.end.bias.copy_(f["end"][1])
        inv.conv.weight.copy_(torch.linalg.inv(f["winv"].double())[..., None])
    for m in [*wn.in_layers, *wn.cond_layers, *wn.res_skip_layers]:
        m.register_forward_pre_hook(lambda mod, args: (qa(args[0]).double(),))
    return wn, inv


def skip_sum(wn, a0, spect):
    """WN's skip sum before `end` (the input of wn.end)"""
    got = []
    h = wn.end.register_forward_hook(lambda mod, args, out: got.append(args[0]))
    wn(a0, spect)
    h.remove()
    return got[0]


def tail(wn, inv, audio, skip):
    """end, the affine coupling and convinv.infer, as WaveGlow.infer does them, on audio [1, c, n] and skip [1, C, n]"""
    h = audio.shape[1] // 2
    out = wn.end(skip)
    s, b = out[:, h:], out[:, :h]
    return inv.infer(torch.cat([audio[:, :h], (audio[:, h:] - b) / torch.exp(s)], 1))


def tail_bound(wn, inv, audio, skip, tskip):
    """the magnitude bound of tail(): sum |term| through end, |audio_1 - b| / exp(s) + |y| |s| terms, |W^-1|"""
    h = audio.shape[1] // 2
    out = wn.end(skip)
    tout = F.conv1d(tskip, wn.end.weight.abs(), wn.end.bias.abs())
    s, b = out[:, h:], out[:, :h]
    y = (audio[:, h:] - b) / torch.exp(s)
    ty = (audio[:, h:].abs() + tout[:, :h]) / torch.exp(s) + y.abs() * (tout[:, h:] + 1)
    winv = inv.conv.weight.squeeze(2).inverse().abs()
    return F.conv1d(torch.cat([audio[:, :h].abs(), ty], 1), winv[..., None])


def wn_bound(wn, a0, spect):
    """the summed |terms| of the skip sum's own GEMMs: sum over the layers of |W_skip| |acts| + |b_skip|, acts exact.
    (Carrying |W| |x| through all eight layers bounds the error strictly but grows by ~sqrt(C) per convolution, to 1e8
    times the values; rounding upstream reaches the skip sum through the network's own gains, which the measured gates
    take in.)"""
    absconv = lambda m, v: F.conv1d(v, m.weight.abs(), m.bias.abs())
    C = wn.n_channels
    x = wn.start(a0)
    tsk = None
    for i in range(N_LAYERS):
        ia = wn.in_layers[i](x) + wn.cond_layers[i](spect)
        acts = torch.tanh(ia[:, :C]) * torch.sigmoid(ia[:, C:])
        rs, trs = wn.res_skip_layers[i](acts), absconv(wn.res_skip_layers[i], acts.abs())
        if i < N_LAYERS - 1:
            x = rs[:, :C] + x
            trs = trs[:, C:]
        tsk = trs if tsk is None else tsk + trs
    return tsk


def per_utterance(lens, Ls, fn, width, dtype=torch.float64):
    """fn(b, n) -> [n, width] per utterance with lens[b] = n > 0, zeros elsewhere: [B, Ls, width]"""
    out = torch.zeros(len(lens), Ls, width, dtype=dtype, device=DEV)
    for b, n in enumerate(lens):
        if n:
            out[b, :n] = fn(b, n)
    return out


def flow_reference(ts, k, C, cond, state, lens, label):
    """float64 (wn skip sum, new state columns o .. 7) of flow k per utterance, with `label`'s operand rounding"""
    c = flow_channels(k)
    o = 8 - c
    wn, inv = oracle_flow(ts, k, C, *operands(label))
    B, Ls, _ = state.shape
    sk, st = torch.zeros(B, Ls, C, dtype=torch.float64, device=DEV), torch.zeros(B, Ls, c, dtype=torch.float64, device=DEV)
    with torch.no_grad():
        for b, n in enumerate(lens):
            if n:
                audio, spect = state[b, :n, o:].double().T[None], cond[b, :n].double().T[None]
                s = skip_sum(wn, audio[:, : c // 2], spect)
                sk[b, :n], st[b, :n] = s[0].T, tail(wn, inv, audio, s)[0].T
    return sk, st


def flow_bound(ts, k, C, cond, state, lens):
    c = flow_channels(k)
    o = 8 - c
    wn, inv = oracle_flow(ts, k, C, *operands("exact"))
    B, Ls, _ = state.shape
    tsk, tst = torch.zeros(B, Ls, C, dtype=torch.float64, device=DEV), torch.zeros(B, Ls, c, dtype=torch.float64, device=DEV)
    with torch.no_grad():
        for b, n in enumerate(lens):
            if n:
                audio, spect = state[b, :n, o:].double().T[None], cond[b, :n].double().T[None]
                s = skip_sum(wn, audio[:, : c // 2], spect)
                tsk[b, :n] = wn_bound(wn, audio[:, : c // 2], spect)[0].T
                tst[b, :n] = tail_bound(wn, inv, audio, s, s.abs())[0].T
    return tsk, tst


def upsample_reference(ts, mels, olens, qa=lambda v: v, qw=lambda w: w, absolute=False):
    """the oracle's upsampling as `infer` runs it (ConvTranspose1d, trim to n * 256 samples, group by 8) per utterance,
    as cond rows [B, L * 32, 640]; absolute: the magnitude bound (|w|, |mel|, |b|)"""
    with torch.device(DEV):
        g = O.WaveGlow(8).double()               # the WNs are not used: the smallest width keeps it cheap
    with torch.no_grad():
        g.upsample.weight.copy_(qw(ts[0]).abs() if absolute else qw(ts[0]))
        g.upsample.bias.copy_(ts[1].abs() if absolute else ts[1])

        def one(b, n):
            m = qa(mels[b, : n // STEPS]).double()
            return g._cond((m.abs() if absolute else m).T[None], n)[0].T
        return per_utterance([v * STEPS for v in olens], mels.shape[1] * STEPS, one, COND)


def rel_error(got, want, bound, mask):
    e = ((got.double() - want).abs() / bound.clamp_min(1e-30))[mask]
    return (float(e.max()), float(e.mean())) if e.numel() else (0.0, 0.0)


def check(gates, mode, got, ref, bound, mask, what):
    """every gate of the mode; returns {label: (max, mean)}"""
    failed, seen = [], {}
    for label, (gmax, gmean) in gates[mode].items():
        mx, mn = rel_error(got, ref(label), bound, mask)
        seen[label] = (mx, mn)
        print(f"GATE {mode:5s} {what:28s} {label:14s} max {mx:.3e} / {gmax:.1e}  mean {mn:.3e} / {gmean:.1e}")
        if not (mx <= gmax and mn <= gmean):
            failed.append((label, mx, mn))
    assert not failed, (mode, what, failed)
    return seen


def valid(lens, Ls):
    return torch.arange(Ls, device=DEV)[None, :] < torch.as_tensor(lens, device=DEV)[:, None]


def flow_inputs(C, k, lens, Ls, seed):
    """seeded cond rows ~ N(0, 0.3^2), state ~ N(0, 1), skip ~ N(0, 0.4^2): values on every row, NaN-free.  With the
    weights of weights(), the couplings are moderate: mean |log s| ~ 0.3, as in tests/test_gpu_waveglow.py"""
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(f"{C}-{k}-{Ls}-{seed}".encode()))
    B = len(lens)
    return (torch.randn(B, Ls, COND, generator=gen, device=DEV) * 0.3, torch.randn(B, Ls, 8, generator=gen, device=DEV),
            torch.randn(B, Ls, C, generator=gen, device=DEV) * 0.4, torch.tensor(lens, dtype=torch.int64, device=DEV))


def check_log_s(ts, k, skip, mask, what):
    """the mean |log s| of flow k's coupling on the skip sums [B, Ls, C] (float64): moderate, neither the identity nor
    a coupling that amplifies by e^3"""
    f = flow_tensors(ts, k)
    h = flow_channels(k) // 2
    log_s = (skip.double() @ f["end"][0][:, :, 0].T.double() + f["end"][1].double())[..., h:][mask]
    m = float(log_s.abs().mean())
    print(f"COUPLING {what:28s} mean |log s| {m:.3f}  max {float(log_s.abs().max()):.3f}")
    assert 0.1 <= m <= 0.8, (what, m)


def nan_past(t, lens):
    return t.masked_fill(~valid(lens, t.shape[1])[..., None], float("nan"))


# ---- the entries are the vocoder -----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_entries_compose_to_the_vocoder_bit_for_bit(mode):
    """upsample, then flows 11 .. 0 in place on the state fp32(z), is fs2_waveglow's audio (sigma = 1, the same z)"""
    C = 256
    n = net(C, mode)
    lib = _lib.load()
    olens = [9, 1, 4, 6]
    B, L = len(olens), max(olens)
    gen = torch.Generator(device=DEV).manual_seed(17)
    mels = torch.randn(B, L, 80, generator=gen, device=DEV) * 2 - 6
    z = torch.randn(B, 8, L * STEPS, generator=gen, device=DEV)
    ol = torch.tensor(olens, dtype=torch.int64, device=DEV)
    import ctypes as Ct
    size = Ct.c_size_t()
    _lib.check(lib.fs2_waveglow_workspace_bytes(n.h, B, L, Ct.byref(size)), "fs2_waveglow_workspace_bytes")
    ws = torch.empty(size.value, dtype=torch.uint8, device=DEV)
    audio = torch.empty(B, L * HOP, device=DEV)
    status = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    _lib.check(lib.fs2_waveglow(n.h, _lib.ptr(mels), _lib.ptr(ol), B, L, 1.0, None, _lib.ptr(z), _lib.ptr(audio), _lib.ptr(status),
                                _lib.ptr(ws), ws.numel(), _lib.stream_ptr(torch.device(DEV))), "fs2_waveglow")
    torch.cuda.synchronize()
    assert int(status.item()) == 0

    cond, _, st = run_upsample(n, mels, ol, planes=False)
    assert st == 0
    steps = ol * STEPS
    state = z.transpose(1, 2).masked_fill(~valid(steps, L * STEPS)[..., None], 0.0).contiguous()
    g = Guarded(B * L * STEPS * 8, torch.float32)
    g.view.copy_(state.reshape(-1))
    for k in reversed(range(N_FLOWS)):
        _, _, st = run_flow(n, k, cond, g.view.view(B, L * STEPS, 8), steps, out=g, wn=False)
        assert st == 0, k
    assert torch.equal(bits(g.view.view(B, L * HOP)), bits(audio)), mode


# ---- the flow kernel alone -----------------------------------------------------------------------------------------
TAIL_CASES = [(C, k) for C in TAIL_CS for k in FLOWS]


@pytest.mark.gpu
@pytest.mark.parametrize("C,k", TAIL_CASES, ids=[f"C{C}-k{k}" for C, k in TAIL_CASES])
def test_flow_kernel_vs_float64(C, k):
    """end conv + coupling + W^-1 on given skip sums: a few fp32 ulps of the summed |terms|, the same bits in every
    mode, in place and out of place; columns < 8 - c keep their sentinels, rows past lens are +0, NaN there is inert"""
    ts, _ = model(C)
    c = flow_channels(k)
    o = 8 - c
    _, state, skip, lens = flow_inputs(C, k, LENS, LS, 1)
    mask = valid(LENS, LS)
    outs = {}
    for mode in MODES:
        n = net(C, mode)
        out, _, st = run_flow(n, k, None, state, lens, skip_in=skip)
        assert st == 0
        ob = bits(out)
        assert bool((ob[..., :o] == 0x7FA5A5A5).all()), "a column < 8 - c was written"
        assert bool((ob[..., o:][~mask] == 0).all()), "rows past lens are not +0"
        inplace, _, _ = run_flow(n, k, None, state, lens, skip_in=skip, out="inplace")
        assert torch.equal(bits(inplace[..., o:]), ob[..., o:]) and torch.equal(bits(inplace[..., :o]), bits(state[..., :o]))
        nan_out, _, _ = run_flow(n, k, None, nan_past(state, LENS), lens, skip_in=nan_past(skip, LENS))
        assert torch.equal(bits(nan_out), ob), "NaN past lens reached the output"
        outs[mode] = out
    for mode in MODES[1:]:
        assert torch.equal(bits(outs[mode]), bits(outs["fp32"])), f"{mode}: the flow kernel is not the same in every mode"
    wn, inv = oracle_flow(ts, k, C, *operands("exact"))
    with torch.no_grad():
        ref = per_utterance(LENS, LS, lambda b, n: tail(wn, inv, state[b, :n, o:].double().T[None], skip[b, :n].double().T[None])[0].T, c)
        bound = per_utterance(LENS, LS, lambda b, n: tail_bound(wn, inv, state[b, :n, o:].double().T[None], skip[b, :n].double().T[None],
                                                                skip[b, :n].double().abs().T[None])[0].T, c)
    check_log_s(ts, k, skip, mask, f"tail C{C} c{c}")
    check({"fp32": GATES["tail"]}, "fp32", outs["fp32"][..., o:], lambda label: ref, bound, mask, f"tail C{C} c{c}")


# ---- a whole flow --------------------------------------------------------------------------------------------------
WN_CASES = [(C, k, mode) for C in WN_CS for k in FLOWS for mode in MODES]


def check_flow(C, k, mode, lens, Ls, seed, what):
    ts, _ = model(C)
    n = net(C, mode)
    c = flow_channels(k)
    o = 8 - c
    cond, state, _, lt = flow_inputs(C, k, lens, Ls, seed)
    mask = valid(lens, Ls)
    out, wn, st = run_flow(n, k, cond, state, lt)
    assert st == 0
    assert bool((bits(out[..., :o]) == 0x7FA5A5A5).all()), "a column < 8 - c was written"
    assert bool((bits(out[..., o:])[~mask] == 0).all()) and bool((bits(wn)[~mask] == 0).all()), "rows past lens are not +0"
    tsk, tst = flow_bound(ts, k, C, cond, state, lens)
    refs = {}

    def ref(label):
        if label not in refs:
            refs[label] = flow_reference(ts, k, C, cond, state, lens, label)
        return refs[label]
    check_log_s(ts, k, ref("exact")[0], mask, f"{what} {mode}")
    seen = check(GATES["wn"], mode, wn, lambda label: ref(label)[0], tsk, mask, f"{what} wn")
    check(GATES["state"], mode, out[..., o:], lambda label: ref(label)[1], tst, mask, f"{what} state")
    if mode in ("f16", "tf32"):           # the fp32-class gates would catch this mode's rounding
        assert seen["exact"][0] > GATES["wn"]["3xf16"]["exact"][0], "the fp32-class gate does not separate the modes"
    return out, wn


@pytest.mark.gpu
@pytest.mark.parametrize("C,k,mode", WN_CASES, ids=[f"C{C}-k{k}-{m}" for C, k, m in WN_CASES])
def test_flow_vs_float64(C, k, mode):
    check_flow(C, k, mode, LENS, LS, 2, f"C{C} k{k}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_flow_vs_float64_past_two_waves_of_tiles(mode):
    """B * Ls = 36,000 step rows: 282 row tiles of the in-layer GEMM, 273 of them live (the rest dead tiles past
    lens), more than 2 x 132, so persistent CTAs walk several tiles each and both consumer warpgroups take tiles"""
    B, Ls = BIG
    check_flow(256, 7, mode, BIG_LENS, Ls, 3, "C256 k7 big")


# ---- the upsampling ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_upsample_vs_float64(mode):
    C = 64
    ts, _ = model(C)
    n = net(C, mode)
    gen = torch.Generator(device=DEV).manual_seed(23)
    B = len(UP_OLENS)
    mels = torch.randn(B, UP_L, 80, generator=gen, device=DEV) * 2 - 6
    ol = torch.tensor(UP_OLENS, dtype=torch.int64, device=DEV)
    cond, planes, st = run_upsample(n, mels, ol)
    assert st == 0
    steps = [v * STEPS for v in UP_OLENS]
    mask = valid(steps, UP_L * STEPS)
    assert bool((bits(cond)[~mask] == 0).all()), "cond rows past olens * 32 are not +0"
    nan_mels = nan_past(mels, UP_OLENS)
    cond_n, planes_n, _ = run_upsample(n, nan_mels, ol)
    assert torch.equal(bits(cond_n), bits(cond)), "NaN in frames past olens reached cond"
    if planes is not None:
        assert torch.equal(bits(planes_n), bits(planes))
        P = 2 if mode == "3xf16" else 1
        sp = split_planes(cond, P).view(torch.float16).float()
        want = (sp[0] + (sp[1] if P == 2 else 0)) * (1 / 16)
        assert torch.equal(bits(planes[mask]), bits(want[mask])), "planes are not split_pair's"
        assert bool((bits(planes)[~mask] == 0).all())
    bound = upsample_reference(ts, mels, UP_OLENS, absolute=True)
    check(GATES["upsample"], mode, cond, lambda label: upsample_reference(ts, mels, UP_OLENS, *operands(label)), bound, mask, "upsample")


# ---- per utterance, bad lengths, range -----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_per_utterance_bits(mode):
    """an utterance alone (Ls = its own length), inside the batch and inside the reversed batch: the same bits, for the
    whole flow and for the upsampling"""
    C, k = 320, 7
    n = net(C, mode)
    lens = [v for v in LENS if v]
    cond, state, _, lt = flow_inputs(C, k, lens, LS, 4)
    out, wn, _ = run_flow(n, k, cond, state, lt)
    rout, rwn, _ = run_flow(n, k, cond.flip(0).contiguous(), state.flip(0).contiguous(), lt.flip(0).contiguous())
    nout, nwn, _ = run_flow(n, k, cond, nan_past(state, lens), lt)
    assert torch.equal(bits(nout), bits(out)) and torch.equal(bits(nwn), bits(wn)), "NaN past lens in state_in reached the output"
    B = len(lens)
    for b, L in enumerate(lens):
        one, one_wn, _ = run_flow(n, k, cond[b: b + 1, :L].contiguous(), state[b: b + 1, :L].contiguous(), lt[b: b + 1])
        for o_, w_ in ((out[b], wn[b]), (rout[B - 1 - b], rwn[B - 1 - b])):
            assert torch.equal(bits(o_[:L]), bits(one[0])) and torch.equal(bits(w_[:L]), bits(one_wn[0])), (mode, b)
    gen = torch.Generator(device=DEV).manual_seed(29)
    olens = [v for v in UP_OLENS if v]
    mels = torch.randn(len(olens), UP_L, 80, generator=gen, device=DEV) * 2 - 6
    ol = torch.tensor(olens, dtype=torch.int64, device=DEV)
    cond, _, _ = run_upsample(n, mels, ol)
    rcond, _, _ = run_upsample(n, mels.flip(0).contiguous(), ol.flip(0).contiguous())
    for b, L in enumerate(olens):
        one, _, _ = run_upsample(n, mels[b: b + 1, :L].contiguous(), ol[b: b + 1])
        assert torch.equal(bits(cond[b, : L * STEPS]), bits(one[0])), (mode, b)
        assert torch.equal(bits(rcond[len(olens) - 1 - b, : L * STEPS]), bits(one[0])), (mode, b)


@pytest.mark.gpu
def test_bad_lengths_are_zero_and_reported():
    """a length outside [0, L] counts as 0 (its rows +0, never read) and sets FS2_WAVEGLOW_BAD_LENGTH; the other
    utterances keep their bits"""
    n = net(64, "3xf16")
    lens = [40, 31, 129]
    cond, state, skip, lt = flow_inputs(64, 7, lens, 130, 5)
    good, good_wn, st = run_flow(n, 7, cond, state, lt)
    assert st == 0
    for bad in (-1, 131, 2 ** 40):
        lb = lt.clone()
        lb[1] = bad
        out, wn, st = run_flow(n, 7, cond, state, lb)
        assert st == BAD_LENGTH
        assert bool((bits(out[1, :, 2:]) == 0).all()) and bool((bits(wn[1]) == 0).all())
        for b in (0, 2):
            assert torch.equal(bits(out[b]), bits(good[b])) and torch.equal(bits(wn[b]), bits(good_wn[b]))
        tail_out, _, st = run_flow(n, 7, None, state, lb, skip_in=skip)
        assert st == BAD_LENGTH and bool((bits(tail_out[1, :, 2:]) == 0).all())
    mels = torch.randn(3, 5, 80, device=DEV) - 6
    cond, _, st = run_upsample(n, mels, torch.tensor([5, 6, 2], device=DEV))
    assert st == BAD_LENGTH and bool((bits(cond[1]) == 0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_range_bit(mode):
    """a start weight x 1e5 (x far past 4094), cond values near 1e4, or mels near 1e4: FS2_WAVEGLOW_RANGE in f16 / 3xf16,
    never in fp32 / tf32"""
    C, k = 64, 11
    want = RANGE if mode in ("f16", "3xf16") else 0
    ts, _ = model(C)
    lens = [40, 0, 9]
    cond, state, _, lt = flow_inputs(C, k, lens, 40, 6)
    n = net(C, mode)
    assert run_flow(n, k, cond, state, lt)[2] == 0
    loud = cond.clone()
    loud[2, :9] = 1e4
    assert run_flow(n, k, loud, state, lt)[2] == want
    mels = torch.randn(2, 6, 80, device=DEV) - 6
    ol = torch.tensor([6, 3], device=DEV)
    assert run_upsample(n, mels, ol)[2] == 0
    mels[1, 2] = 1e4
    assert run_upsample(n, mels, ol)[2] == want
    big = list(ts)
    base = 2 + k * PER_FLOW
    big[base] = ts[base] * 1e5
    assert run_flow(Net(C, mode, big), k, cond, state, lt)[2] == want


@pytest.mark.gpu
def test_refusals_that_need_a_handle():
    """an unloaded handle, and fs2_waveglow's row limits on B * L step rows, are refused before any launch"""
    import ctypes as Ct
    lib = _lib.load()
    h = Ct.c_void_p()
    _lib.check(lib.fs2_waveglow_create(Ct.byref(h), MODE["fp32"], 64), "fs2_waveglow_create")
    p = torch.zeros(64, device=DEV)
    nets = {mode: net(64, mode) for mode in ("fp32", "3xf16")}      # loading launches kernels: before the count starts
    before = lib.fs2_kernel_launches()
    try:
        assert lib.fs2_op_waveglow_flow(h.value, 0, _lib.ptr(p), None, _lib.ptr(p), _lib.ptr(p), _lib.ptr(p), 1, 1, None, _lib.ptr(p), None) == -1
        assert b"unloaded" in lib.fs2_last_error()
        assert lib.fs2_op_waveglow_upsample(h.value, _lib.ptr(p), _lib.ptr(p), 1, 1, _lib.ptr(p), None, _lib.ptr(p), None) == -1
        assert b"unloaded" in lib.fs2_last_error()
    finally:
        lib.fs2_waveglow_destroy(h.value)
    # fp32: one past 65535 * 128 rows; the plane modes: 2^31 rows
    for mode, B, Ls in (("fp32", 1, 65535 * 128 + 1), ("3xf16", 2, 2 ** 30)):
        n = nets[mode]
        assert lib.fs2_op_waveglow_flow(n.h, 0, _lib.ptr(p), None, _lib.ptr(p), _lib.ptr(p), _lib.ptr(p), B, Ls, None, _lib.ptr(p),
                                        None) == -1, mode
        assert b"rows exceed" in lib.fs2_last_error()
        assert lib.fs2_op_waveglow_upsample(n.h, _lib.ptr(p), _lib.ptr(p), B, -(-Ls // STEPS), _lib.ptr(p), None, _lib.ptr(p),
                                            None) == -1, mode
        assert b"rows exceed" in lib.fs2_last_error()
        if mode == "fp32":
            assert lib.fs2_op_waveglow_upsample(n.h, _lib.ptr(p), _lib.ptr(p), 1, 1, _lib.ptr(p), _lib.ptr(p), _lib.ptr(p), None) == -1
            assert b"cond_planes" in lib.fs2_last_error()
    assert lib.fs2_kernel_launches() == before
