"""The fused optimizer without a GPU (DESIGN.md §15): the C entries in the header, the library and _lib, the workspace size
against the plan in _optim_plan.py, argument checks (fake pointers, never dereferenced), the Noam / Adam scalar
restatement against the reference's NoamOpt.rate for steps 1 .. 10^6, NoamAdam's refusals and state_dict layout, the
drop-in hook and the kernels' build report."""
import ctypes as C
import glob
import importlib.util
import os
import re
import sys
import types

import numpy as np
import pytest
import torch

import _optim_plan as P
from fastspeech2_b200 import FeedForwardTransformer, _lib
from fastspeech2_b200 import dropin_run
from fastspeech2_b200 import optim as O
from fastspeech2_b200.hparams import load_hp

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_OPT = os.path.join(REPO, "oracle", "_ref", "core", "optimizer.py")
ENTRIES = ("fs2_optim_ws_bytes", "fs2_optim_noam_adam", "fs2_optim_clip_noam_adam", "fs2_optim_noam_scalars")
FAKE = 1 << 20
FS2_ERR_INVALID = -1


def ref_optimizer():
    if not os.path.isfile(REF_OPT):
        pytest.skip("reference not staged in oracle/_ref")
    spec = importlib.util.spec_from_file_location("ref_core_optimizer", REF_OPT)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def lib_ws(numel):
    arr = (C.c_int64 * max(1, len(numel)))(*numel)
    n = C.c_size_t(0)
    rc = _lib.load().fs2_optim_ws_bytes(arr, len(numel), C.byref(n))
    return rc, int(n.value)


def model_numels():
    return [p.numel() for p in FeedForwardTransformer(68, 80, load_hp()).parameters()]


# ---- interface and workspace ------------------------------------------------------------------------------------------------------
def test_entries_are_exported_and_declared():
    lib = _lib.load()
    hdr = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    for name in ENTRIES:
        assert name in _lib.SIGNATURES and hasattr(lib, name)
        assert re.search(rf"\bint {name}\(", hdr), name
    assert f"#define FS2_OPTIM_CHUNK {P.CHUNK}" in hdr and _lib.FS2_OPTIM_CHUNK == P.CHUNK
    assert "align256(8 n_chunks) + align256(8 n) + align256(16)" in hdr


@pytest.mark.parametrize("numel", [[1], [3], [P.CHUNK - 1], [P.CHUNK], [P.CHUNK + 1], [1, 3, P.CHUNK + 1, 2 * P.CHUNK - 1],
                                   "model"])
def test_workspace_matches_the_plan(numel):
    if numel == "model":
        numel = model_numels()
        assert sum(numel) > 30_000_000
    assert lib_ws(numel) == (0, P.ws_bytes(numel))


def test_chunk_plan():
    counts, first, total = P.chunks([1, P.CHUNK, P.CHUNK + 1, 3])
    assert counts == [1, 1, 2, 1] and first == [0, 1, 2, 4] and total == 5


@pytest.mark.parametrize("numel", [[], [0], [5, 0], [-1], [1 << 62, 1 << 62], [(1 << 46)] * 2])
def test_bad_tables_are_invalid(numel):
    assert lib_ws(numel)[0] == FS2_ERR_INVALID


def _hp():
    return _lib.NoamAdamHp(*P.noam_constants(384, 1.0, 4000), 0.9, 0.98, 1e-9)


def test_step_entries_refuse_bad_arguments():
    lib = _lib.load()
    numel = (C.c_int64 * 2)(5, P.CHUNK + 3)
    need = P.ws_bytes([5, P.CHUNK + 3])
    hp = _hp()
    ok = dict(table=FAKE, numel=numel, n=2, hp=hp, step=FAKE, lr=FAKE, ws=FAKE, ws_bytes=need)

    def plain(**kw):
        a = dict(ok, **kw)
        return lib.fs2_optim_noam_adam(a["table"], a["numel"], a["n"], a["hp"], a["step"], a["lr"], a["ws"], a["ws_bytes"], None)

    def clip(norm=FAKE, **kw):
        a = dict(ok, **kw)
        return lib.fs2_optim_clip_noam_adam(a["table"], a["numel"], a["n"], a["hp"], 1.0, a["step"], a["lr"], norm, a["ws"],
                                            a["ws_bytes"], None)

    for call in (plain, clip):
        assert call(n=0) == FS2_ERR_INVALID
        assert call(numel=(C.c_int64 * 2)(5, 0)) == FS2_ERR_INVALID
        assert call(ws_bytes=need - 1) == FS2_ERR_INVALID and b"needed" in lib.fs2_last_error()
        assert call(ws=FAKE + 8) == FS2_ERR_INVALID
        for k in ("table", "step", "lr", "ws"):
            assert call(**{k: None}) == FS2_ERR_INVALID
        assert call(hp=None) == FS2_ERR_INVALID
    assert clip(norm=None) == FS2_ERR_INVALID
    assert lib.fs2_optim_noam_scalars(0, 4, hp, FAKE, FAKE, FAKE, None) == FS2_ERR_INVALID
    assert lib.fs2_optim_noam_scalars(1, 0, hp, FAKE, FAKE, FAKE, None) == FS2_ERR_INVALID


# ---- scalar restatement against the reference -------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", [(384, 1.0, 4000), (256, 1.0, 4), (384, 2.0, 4)])
def test_rate_restatement_matches_noamopt(cfg):
    R = ref_optimizer()
    d, f, w = cfg
    ref = R.NoamOpt(d, f, w, None)
    n = 10 ** 6
    steps = np.arange(1, n + 1)
    py_lr = np.array([ref.rate(s) for s in range(1, n + 1)])
    lr = P.noam_rate(steps, d, f, w)
    # the restatement rounds step ** -0.5 correctly; libm's pow does not always: one ulp apart at some steps ...
    assert np.all(np.abs(lr - py_lr) <= 2 * np.spacing(py_lr))
    assert np.mean(lr != py_lr) < 1e-3
    # ... and never in what torch's Adam consumes: the fp32 step size and bias-correction root
    ss, bc = P.adam_scalars(steps, lr)
    want_ss = np.array([(l / (1 - 0.9 ** float(s))) * -1 for s, l in zip(range(1, n + 1), py_lr)]).astype(np.float32)
    want_bc = np.array([(1 - 0.98 ** float(s)) ** 0.5 for s in range(1, n + 1)]).astype(np.float32)
    assert np.array_equal(ss, want_ss) and np.array_equal(bc, want_bc)


def test_rsqrt_is_correctly_rounded():
    from decimal import Decimal, getcontext
    getcontext().prec = 50
    for s in (2, 3, 1769, 2397, 4000, 99991, 10 ** 6 - 1):
        y = float(P.rsqrt(np.array([float(s)]))[0])
        exact = Decimal(1) / Decimal(s).sqrt()
        for nb in (np.nextafter(y, 0), np.nextafter(y, 1)):
            assert abs(Decimal(y) - exact) < abs(Decimal(float(nb)) - exact), s


# ---- NoamAdam on the host -----------------------------------------------------------------------------------------------------------
def test_refusals():
    with pytest.raises(ValueError, match="no trainable"):
        O.NoamAdam([], 384, 1.0, 4000)
    with pytest.raises(ValueError, match="no trainable"):
        O.NoamAdam([torch.zeros(3)], 384, 1.0, 4000)
    with pytest.raises(ValueError, match="CUDA float32"):
        O.NoamAdam([torch.zeros(3, requires_grad=True)], 384, 1.0, 4000)
    with pytest.raises(ValueError, match="CUDA float32"):
        O.get_std_opt(FeedForwardTransformer(68, 80, load_hp()), 384, 4000, 1.0)
    with pytest.raises(ValueError, match="groups"):
        O.NoamAdam([{"params": [torch.zeros(3, requires_grad=True)]}], 384, 1.0, 4000)


def test_state_dict_layout_is_noamopt_over_torch_adam(monkeypatch):
    """Key for key the reference's NoamOpt over torch's Adam, with a CPU Adam's state loaded (the CUDA check waived: no
    kernel runs here)."""
    R = ref_optimizer()
    monkeypatch.setattr(O, "_require_cuda", lambda params: None)
    torch.manual_seed(0)
    a = [torch.randn(4, 3, requires_grad=True), torch.randn(5, requires_grad=True), torch.randn(2, requires_grad=True)]
    b = [p.detach().clone().requires_grad_() for p in a]
    ref = R.get_std_opt(types.SimpleNamespace(parameters=lambda: iter(a)), 384, 4000, 1.0)
    ours = O.get_std_opt(types.SimpleNamespace(parameters=lambda: iter(b)), 384, 4000, 1.0)
    e0, o0 = ref.state_dict(), ours.state_dict()
    assert list(e0) == list(o0) and e0["optimizer"] == o0["optimizer"]
    for s in range(3):
        for p in a[:2]:
            p.grad = torch.randn_like(p)
        ref.step()
    want = ref.state_dict()
    ours.load_state_dict(want)
    got = ours.state_dict()
    assert list(got) == list(want)
    assert {k: got[k] for k in got if k != "optimizer"} == {k: want[k] for k in want if k != "optimizer"}
    assert got["optimizer"]["param_groups"] == want["optimizer"]["param_groups"]
    assert sorted(got["optimizer"]["state"]) == sorted(want["optimizer"]["state"]) == [0, 1]
    for i, st in want["optimizer"]["state"].items():
        assert list(got["optimizer"]["state"][i]) == list(st)
        for k, v in st.items():
            w = got["optimizer"]["state"][i][k]
            assert (w.dtype, w.device, w.shape) == (v.dtype, v.device, v.shape) and torch.equal(w, v), (i, k)
    assert ours.rate(7) == ref.rate(7)


# ---- drop-in hook ------------------------------------------------------------------------------------------------------------------
def _fake_checkout(tmp_path):
    core = tmp_path / "core"
    core.mkdir()
    (core / "__init__.py").write_text("")
    (core / "optimizer.py").write_text("def get_std_opt(model, d_model, warmup, factor):\n    return 'reference'\n")
    (tmp_path / "train_fastspeech.py").write_text(
        "from core.optimizer import get_std_opt\nimport builtins\nbuiltins._fs2_test_opt = get_std_opt\n")
    return str(tmp_path / "train_fastspeech.py")


@pytest.mark.parametrize("env", [None, "torch", "fused"])
def test_dropin_hook_replaces_get_std_opt_only_when_asked(env, tmp_path, monkeypatch):
    import builtins
    script = _fake_checkout(tmp_path)
    saved_path, saved_argv = list(sys.path), list(sys.argv)
    for k in [k for k in sys.modules if k == "core" or k.startswith("core.")]:
        monkeypatch.delitem(sys.modules, k)
    if env is None:
        monkeypatch.delenv(dropin_run.OPTIMIZER_ENV, raising=False)
    else:
        monkeypatch.setenv(dropin_run.OPTIMIZER_ENV, env)
    try:
        dropin_run.main([script])
        fn = builtins._fs2_test_opt
    finally:
        sys.path[:], sys.argv[:] = saved_path, saved_argv
        for k in [k for k in sys.modules if k == "core" or k.startswith("core.")]:
            del sys.modules[k]
        builtins.__dict__.pop("_fs2_test_opt", None)
    assert (fn is O.get_std_opt) == (env == "fused")
    if env != "fused":
        assert fn(None, 1, 1, 1) == "reference"


def test_dropin_refuses_unknown_optimizer(tmp_path, monkeypatch):
    monkeypatch.setenv(dropin_run.OPTIMIZER_ENV, "adamw")
    saved_path, saved_argv = list(sys.path), list(sys.argv)
    try:
        with pytest.raises(SystemExit, match="FS2_OPTIMIZER"):
            dropin_run.main([_fake_checkout(tmp_path)])
    finally:
        sys.path[:], sys.argv[:] = saved_path, saved_argv


# ---- build report ---------------------------------------------------------------------------------------------------------------------
def test_optim_kernels_do_not_spill():
    reports = glob.glob(os.path.join(REPO, "fastspeech2_b200", "build", "optim.ptxas.txt"))
    if not reports:
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = open(reports[0]).read()
    props = re.findall(r"Function properties for (\S*optim_\w+kernel\S*)\n(.*)", text)
    names = {re.search(r"\d(optim_[a-z_]+_kernel)E", n).group(1) for n, _ in props}
    assert names == {"optim_sumsq_kernel", "optim_scalar_kernel", "optim_update_kernel", "optim_noam_scalars_kernel"}, names
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)
