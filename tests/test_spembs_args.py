"""External speaker embeddings (DESIGN.md section 27) without a GPU: the oracle against the unmodified reference
(tests/golden/spembs.npz), hp parsing and the checkpoint layout, the argument errors that need no device, the dataset and
collation tuples, `speakers average`, the C header and bindings, and the C entries' refusals before any launch."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from fastspeech2_b200 import FeedForwardTransformer, _lib
from fastspeech2_b200 import data as D
from fastspeech2_b200 import speakers as S
from fastspeech2_b200.hparams import load_hp
from oracle import spemb_oracle as SPO
import _spembs_golden as EG

T = torch.from_numpy
HEADER = os.path.join(os.path.dirname(GOLDEN), "..", "include", "fs2_b200.h")
NEW_ENTRIES = ("fs2_encode_spemb", "fs2_length_plan_cap_spemb", "fs2_op_row_norm_spemb", "fs2_spemb_project",
               "fs2_spemb_project_backward")


def hp_with(d=None, n=0, kind=None):
    hp = load_hp()
    if d is not None:
        hp["model"]["spk_embed_dim"] = d
    if n:
        hp["model"]["n_speakers"] = n
    if kind is not None:
        hp["model"]["spk_embed_integration_type"] = kind
    return hp


def close(a, b, tol=1e-6):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.max(np.abs(a - b)) <= tol, float(np.max(np.abs(a - b)))


# ---- the oracle against the reference -------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", EG.CONFIGS)
def test_spemb_oracle_matches_reference(golden, weights, cfg):
    g = golden("spembs")
    c = EG.cfg(g, cfg)
    e, W, bias = EG.seeded()
    tab = EG.table() if cfg == "both" else None
    spk = T(g["speakers"])
    torch.set_num_threads(1)
    with torch.no_grad():
        b, a, d, eo, po = SPO.forward_path(weights, tab, spk, W, bias, e, T(g["xs"]), T(g["ilens"]), T(g["olens"]),
                                           T(g["ds"]).clone(), T(g["es"]), T(g["ps"]), False)
        close(d, c["tf_d_outs"]); close(eo, c["tf_e_outs"]); close(po, c["tf_p_outs"])
        mels, means = EG.mel_checks(c, "tf", b, a, T(g["olens"]))
        for _, got, want in mels + means:
            close(got, want)
        b, a, d, eh, ph = SPO.forward_path(weights, tab, spk, W, bias, e, T(g["xs"]), T(g["ilens"]), is_inference=True)
    assert torch.equal(d, T(c["inf_d_outs"])) and a.shape[1] == int(c["inf_frames"])
    assert torch.equal(eh.argmax(-1), T(c["inf_e_ids"]).long()) and torch.equal(ph.argmax(-1), T(c["inf_p_ids"]).long())
    mels, means = EG.mel_checks(c, "inf", b, a, d.sum(1))
    for _, got, want in mels + means:
        close(got, want)


def test_golden_inputs_and_gradient_samples_are_regenerated(golden):
    g = golden("spembs")
    EG.batch(g)
    assert int(g["D"]) == EG.D and int(g["n_speakers"]) == 5
    m = FeedForwardTransformer(68, 80, hp_with(EG.D, 5))
    samples = EG.grad_samples(g, {k: v.numel() for k, v in m.named_parameters()})
    assert set(samples) == {k for k, _ in m.named_parameters()} - set(json.loads(str(g["no_grad"])))
    e, _, _ = EG.seeded()
    assert float(e[3].abs().max()) == 0.0 and torch.equal(e[1], e[5])     # a zero-norm embedding, and a shared one


def test_golden_embeddings_matter(golden):
    g = golden("spembs")
    both, emb = EG.cfg(g, "both"), EG.cfg(g, "emb")
    assert not np.array_equal(both["inf_d_outs"], emb["inf_d_outs"])
    assert np.abs(g["grad/spk_embed_proj.bias"]).max() > 0


# ---- hp and the checkpoint layout ------------------------------------------------------------------------------------------
def test_state_dict_keys_and_order():
    ref = json.load(open(os.path.join(GOLDEN, "state_dict_keys.json")))
    for d in (None, 0):
        hp = hp_with()
        hp["model"]["spk_embed_dim"] = d
        m = FeedForwardTransformer(68, 80, hp)
        assert [[k, list(v.shape), str(v.dtype)] for k, v in m.state_dict().items()] == ref and m.spk_embed_dim == 0
    keys = [[k, list(v.shape), str(v.dtype)] for k, v in FeedForwardTransformer(68, 80, hp_with(192)).state_dict().items()]
    assert keys == ref + [["spk_embed_proj.weight", [256, 192], "torch.float32"], ["spk_embed_proj.bias", [256], "torch.float32"]]
    keys = [k for k in FeedForwardTransformer(68, 80, hp_with(512, 3, "add")).state_dict()]
    assert keys[-3:] == ["speaker_embed.weight", "spk_embed_proj.weight", "spk_embed_proj.bias"]


def test_other_parameters_initialise_as_without_embeddings():
    torch.manual_seed(3)
    a = FeedForwardTransformer(68, 80, hp_with(n=4)).state_dict()
    torch.manual_seed(3)
    b = FeedForwardTransformer(68, 80, hp_with(256, 4)).state_dict()
    assert all(torch.equal(a[k], b[k]) for k in a)
    bound = 1 / 256 ** 0.5                                   # nn.Linear's default init: U(-1/sqrt(D), 1/sqrt(D))
    assert float(b["spk_embed_proj.weight"].abs().max()) <= bound and float(b["spk_embed_proj.bias"].abs().max()) <= bound


@pytest.mark.parametrize("hp_kw, match", [
    (dict(d=-1), r"spk_embed_dim must be 0 \(none\) or an int in \[1, 4096\]"),
    (dict(d=4097), r"spk_embed_dim must be 0 \(none\) or an int in \[1, 4096\]"),
    (dict(d=192.0), "spk_embed_dim must be"),
    (dict(d=True), "spk_embed_dim must be"),
    (dict(d=192, kind="concat"), r"spk_embed_integration_type must be one of \['add'\], got 'concat'"),
    (dict(kind="concat"), "spk_embed_integration_type"),
])
def test_bad_hp_is_refused(hp_kw, match):
    with pytest.raises(ValueError, match=match):
        FeedForwardTransformer(68, 80, hp_with(**hp_kw))


@pytest.mark.parametrize("d", [1, 192, 4096])
def test_dims_in_range_are_accepted(d):
    assert FeedForwardTransformer(68, 80, hp_with(d)).spk_embed_proj.weight.shape == (256, d)


def test_from_checkpoint_reads_d(weights):
    with open(os.path.join(os.path.dirname(GOLDEN), "..", "fastspeech2_b200", "configs", "default.yaml")) as fh:
        hp_str = fh.read()                                  # written before the key existed
    sd = dict(weights)
    sd["spk_embed_proj.weight"], sd["spk_embed_proj.bias"] = torch.zeros(256, 320), torch.zeros(256)
    m = FeedForwardTransformer.from_checkpoint({"model": sd, "hp_str": hp_str})
    assert m.spk_embed_dim == 320 and tuple(m.spk_embed_proj.weight.shape) == (256, 320)
    assert FeedForwardTransformer.from_checkpoint({"model": sd, "hp_str": hp_str}, hp=hp_with(320)).spk_embed_dim == 320
    with pytest.raises(ValueError, match="spk_embed_dim = 192 but the checkpoint's spk_embed_proj.weight takes D = 320"):
        FeedForwardTransformer.from_checkpoint({"model": sd, "hp_str": hp_str}, hp=hp_with(192))
    with pytest.raises(ValueError, match="spk_embed_dim = 192 but the checkpoint's spk_embed_proj.weight takes D = 0"):
        FeedForwardTransformer.from_checkpoint({"model": dict(weights), "hp_str": hp_str}, hp=hp_with(192))
    assert FeedForwardTransformer.from_checkpoint({"model": dict(weights), "hp_str": hp_str}).spk_embed_dim == 0


def test_signatures_stay_the_references():
    import inspect
    m = FeedForwardTransformer(68, 80, hp_with(192))
    assert list(inspect.signature(m.forward).parameters) == ["xs", "ilens", "ys", "olens", "ds", "es", "ps"]
    assert list(inspect.signature(m.inference).parameters) == ["x"]


# ---- argument errors that need no device -----------------------------------------------------------------------------------
@pytest.mark.parametrize("d, spembs, match", [
    (192, None, r"the model takes 192-dim speaker embeddings: pass them"),
    (0, torch.zeros(2, 192), r"the model has no projection \(hp.model.spk_embed_dim is 0\)"),
    (192, torch.zeros(2, 192, dtype=torch.float64), "spembs must be a float32 tensor, got torch.float64"),
    (192, np.zeros((2, 192), dtype=np.float32), "spembs must be a float32 tensor"),
    (192, torch.zeros(2, 191), r"spembs must be \[B=2, D=192\], got \(2, 191\)"),
    (192, torch.zeros(3, 192), r"spembs must be \[B=2, D=192\], got \(3, 192\)"),
    (192, torch.zeros(192), r"spembs must be \[B=2, D=192\]"),
    (192, torch.zeros(2, 192, device="meta"), "spembs must be on cpu with the model's input, got meta"),
])
def test_spemb_errors(d, spembs, match):
    m = FeedForwardTransformer(68, 80, hp_with(d)).eval()
    xs, il = torch.ones(2, 5, dtype=torch.int64), torch.tensor([5, 3])
    with pytest.raises(ValueError, match=match):
        m.synthesize(xs, il, spembs=spembs)
    with pytest.raises(ValueError, match=match):
        m._forward(xs, il, is_inference=True, spembs=spembs)


def test_inference_spemb_errors():
    m = FeedForwardTransformer(68, 80, hp_with(16)).eval()
    x = torch.ones(5, dtype=torch.int64)
    with pytest.raises(ValueError, match="pass them"):
        m.inference(x)
    with pytest.raises(ValueError, match=r"spemb must be a \[D\] tensor, got shape \(1, 16\)"):
        m.inference(x, spemb=torch.zeros(1, 16))
    with pytest.raises(ValueError, match=r"spembs must be \[B=1, D=16\], got \(1, 8\)"):
        m.inference_controlled(x, spemb=torch.zeros(8), speed=1.2)
    with pytest.raises(ValueError, match="no projection"):
        FeedForwardTransformer(68, 80, hp_with()).eval().inference(x, spemb=torch.zeros(16))


# ---- data ------------------------------------------------------------------------------------------------------------------
def _item(T_, L, spk=None, emb=None, n_extra=0):
    it = (np.arange(1, T_ + 1), np.ones((L, 80), np.float32), f"u{T_}", L, np.ones(T_, np.int64), np.ones(L, np.float32),
          np.ones(L, np.float32))
    if n_extra >= 1:
        it = it + (spk,)
    if n_extra >= 2:
        it = it + (emb,)
    return it


def test_collation_with_embeddings():
    e = [np.arange(4, dtype=np.float32) + i for i in range(2)]
    plain = [_item(3, 5), _item(2, 4)]
    base = D.collate_tts(plain)
    assert len(base) == 9
    out = D.collate_tts([_item(3, 5, 1, e[0], 2), _item(2, 4, 0, e[1], 2)])
    assert len(out) == 11 and out[9].tolist() == [1, 0] and out[10].dtype == torch.float32
    assert torch.equal(out[10], torch.from_numpy(np.stack(e)))
    assert all(torch.equal(a, b) if torch.is_tensor(a) else a == b for a, b in zip(out[:9], base))
    out = D.collate_tts([_item(3, 5, None, e[0], 2), _item(2, 4, None, e[1], 2)])
    assert len(out) == 11 and out[9] is None and torch.equal(out[10], torch.from_numpy(np.stack(e)))
    with pytest.raises(ValueError, match="all carry a speaker id or all carry None"):
        D.collate_tts([_item(3, 5, 1, e[0], 2), _item(2, 4, None, e[1], 2)])
    with pytest.raises(ValueError, match="one D"):
        D.collate_tts([_item(3, 5, None, e[0], 2), _item(2, 4, None, np.zeros(3, np.float32), 2)])
    with pytest.raises(ValueError, match="all 9"):
        D.collate_tts([_item(3, 5, 1, e[0], 2), _item(2, 4, 0, None, 1)])
    pc = D.PinnedCollator(4, 8, 8, pin=False, spk_embed_dim=4)
    got = pc([_item(3, 5, 1, e[0], 2), _item(2, 4, 0, e[1], 2)])
    assert len(got) == 11 and got[9].tolist() == [1, 0] and torch.equal(got[10], torch.from_numpy(np.stack(e)))
    assert len(pc(plain)) == 9
    with pytest.raises(ValueError, match="D=4, but the collator holds spk_embed_dim=3"):
        D.PinnedCollator(4, 8, 8, pin=False, spk_embed_dim=3)([_item(3, 5, 1, e[0], 2)])


def _tree(tmp_path, wavs):
    (tmp_path / "mels").mkdir(); (tmp_path / "energy").mkdir(); (tmp_path / "pitch").mkdir(); (tmp_path / "spemb").mkdir()
    lines = []
    for i, w in enumerate(wavs):
        stem = w.split(".")[0]
        np.save(tmp_path / "mels" / f"{stem}.npy", np.zeros((80, 6), np.float32))
        np.save(tmp_path / "energy" / f"{stem}.npy", np.ones(6, np.float32))
        np.save(tmp_path / "pitch" / f"{stem}.npy", np.ones(6, np.float32))
        lines.append(f"t|1 3|3 3|AA B|{w}")
    fl = tmp_path / "list.txt"
    fl.write_text("\n".join(lines) + "\n")
    return str(fl)


def test_filelist_dataset_reads_embeddings(tmp_path):
    fl = _tree(tmp_path, ["p1_001.wav", "p2_001.wav"])
    rng = np.random.default_rng(0)
    embs = {s: rng.standard_normal(12).astype(np.float32) for s in ("p1_001", "p2_001")}
    for s, e in embs.items():
        np.save(tmp_path / "spemb" / f"{s}.npy", e)
    syms = ["_", "AA", "B"]
    plain = D.FilelistDataset(fl, str(tmp_path), syms)
    assert len(plain[0]) == 7 and plain.spemb_dim() == 0
    ds = D.FilelistDataset(fl, str(tmp_path), syms, spemb_dir=str(tmp_path / "spemb"))
    it = ds[1]
    assert len(it) == 9 and it[7] is None and it[8].dtype == np.float32 and np.array_equal(it[8], embs["p2_001"])
    assert all(np.array_equal(a, b) if isinstance(a, np.ndarray) else a == b for a, b in zip(it[:7], plain[1]))
    assert ds.spemb_dim() == 12
    ds = D.FilelistDataset(fl, str(tmp_path), syms, speaker_map={"p1": 0, "p2": 1}, spemb_dir=str(tmp_path / "spemb"))
    assert ds[1][7] == 1 and np.array_equal(ds[1][8], embs["p2_001"])
    out = D.collate_tts([ds[0], ds[1]])
    assert out[9].tolist() == [0, 1] and out[10].shape == (2, 12)
    np.save(tmp_path / "spemb" / "p2_001.npy", np.zeros((2, 3), np.float32))
    with pytest.raises(ValueError, match=r"a speaker embedding must be a float \[D\] array"):
        ds[1]


def test_speakers_average_against_numpy(tmp_path):
    wavs = ["p1_001.wav", "p1_002.wav", "p2_001.wav", "p1_003.wav"]
    fl = _tree(tmp_path, wavs)
    rng = np.random.default_rng(1)
    embs = {w.split(".")[0]: (rng.standard_normal(7) * 5).astype(np.float32) for w in wavs}
    embs["p1_003"] = np.zeros(7, np.float32)           # a zero-norm embedding counts as zero
    for s, e in embs.items():
        np.save(tmp_path / "spemb" / f"{s}.npy", e)
    out = tmp_path / "avg"
    S.main(["average", "--filelist", fl, "--spemb-dir", str(tmp_path / "spemb"), "-o", str(out)])
    assert sorted(os.listdir(out)) == ["p1.npy", "p2.npy"]
    unit = lambda v: v.astype(np.float64) / max(np.linalg.norm(v.astype(np.float64)), 1e-12)
    want = {"p1": (unit(embs["p1_001"]) + unit(embs["p1_002"]) + unit(embs["p1_003"])) / 3, "p2": unit(embs["p2_001"])}
    for name, w in want.items():
        got = np.load(out / f"{name}.npy")
        assert got.dtype == np.float32 and got.shape == (7,)
        assert np.max(np.abs(got - w)) <= 1e-7
    np.save(tmp_path / "spemb" / "p2_001.npy", np.array([1.0, np.nan] + [0.0] * 5, np.float32))
    with pytest.raises(ValueError, match="non-finite"):
        S.average(fl, str(tmp_path / "spemb"))


# ---- C header and bindings -------------------------------------------------------------------------------------------------
def _prototypes():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return {m.group(1): m.group(2) for m in re.finditer(r"\bint\s+(fs2_\w+)\s*\(([^)]*)\)\s*;", text)}


@pytest.mark.parametrize("name", NEW_ENTRIES)
def test_header_and_binding_agree(name):
    protos = _prototypes()
    assert name in protos and name in _lib.SIGNATURES
    assert len([a for a in protos[name].split(",") if a.strip()]) == len(_lib.SIGNATURES[name]), name


def test_header_constants():
    text = open(HEADER).read()
    assert re.search(r"#define FS2_SPEMB_NONFINITE 16\b", text) and _lib.FS2_SPEMB_NONFINITE == 16
    assert re.search(r"#define FS2_SPEMB_MAX_DIM 4096\b", text) and _lib.FS2_SPEMB_MAX_DIM == 4096
    bits = [_lib.FS2_PLAN_BAD_ILENS, _lib.FS2_PLAN_BAD_CONTROL, _lib.FS2_PLAN_OVERFLOW, _lib.FS2_PLAN_BAD_SPEAKER]
    assert all(_lib.FS2_SPEMB_NONFINITE & b == 0 for b in bits) and _lib.FS2_SPEMB_NONFINITE < 1 << _lib.FS2_SYNTH_VOC_SHIFT


def test_row_norm_desc_layout_is_unchanged():
    names = [f[0] for f in _lib.RowNormDesc._fields_]
    assert names[-4:] == ["spk_table", "spk", "n_spk", "spk_L"] and "spk_vec" not in names


# ---- refusals before any launch --------------------------------------------------------------------------------------------
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="refusal tests run only where no CUDA device is visible")
A = 0x10000


def _refused(rc, *words):
    msg = _lib.load().fs2_last_error().decode()
    assert rc == -1, (rc, msg)
    for w in words:
        assert w in msg, (w, msg)


@no_device
@pytest.mark.parametrize("args, words", [
    ((0, A, A, 2, 192, 256, A, None, None, None, None), "null argument"),
    ((A, A, A, 2, 192, 256, 0, None, None, None, None), "null argument"),
    ((A, A, A, 2, 0, 256, A, None, None, None, None), "D=0"),
    ((A, A, A, 2, 4097, 256, A, None, None, None, None), "D=4097"),
    ((A, A, A, -1, 192, 256, A, None, None, None, None), "B=-1"),
    ((A, A, A, 2, 192, 0, A, None, None, None, None), "adim=0"),
])
def test_spemb_project_refuses(args, words):
    _refused(_lib.load().fs2_spemb_project(*args), words)


@no_device
@pytest.mark.parametrize("args, words", [
    ((0, A, 2, 192, 256, A, A, None), "null argument"),
    ((A, A, 2, 192, 256, A, 0, None), "null argument"),
    ((A, A, 2, 4097, 256, A, A, None), "D=4097"),
    ((A, A, 2, 192, 0, A, A, None), "adim=0"),
])
def test_spemb_project_backward_refuses(args, words):
    _refused(_lib.load().fs2_spemb_project_backward(*args), words)


@no_device
def test_row_norm_spemb_refuses():
    base = dict(x=A, ldx=256, gamma=A + 0x1000, beta=A + 0x2000, eps=1e-5, rows=8, C=256, out=A + 0x3000, ldo=256)
    d = _lib.RowNormDesc(**base)
    _refused(_lib.load().fs2_op_row_norm_spemb(C.byref(d), A + 0x4000, None), "spk_vec", "spk_L > 0")
    d = _lib.RowNormDesc(**dict(base, spk_L=4))
    _refused(_lib.load().fs2_op_row_norm_spemb(C.byref(d), A + 0x4004, None), "spk_vec must be 16-byte aligned")
    _refused(_lib.load().fs2_op_row_norm_spemb(None, A, None), "null descriptor")


# ---- no floating-point atomics in the new kernels --------------------------------------------------------------------------
def test_spemb_kernels_have_no_float_atomics():
    from test_train_deterministic_args import FLOAT_ATOMIC, RETURNING_INT_ATOMG, sass_functions
    sass = sass_functions()
    for name in ("spemb_project_kernel", "spemb_project_backward_kernel"):
        assert name in sass, sorted(k for k in sass if "spemb" in k)
        assert not FLOAT_ATOMIC.search(sass[name]) and not RETURNING_INT_ATOMG.search(sass[name]), name
