"""The duration aligner without a device (fastspeech2_b200.aligner, DESIGN.md section 24): filelist parsing and writing,
the symbol table, argument and size checks of the C entries and the module, the workspace formula, the kernels'
register report; the oracle's forward-sum against a direct CTC lattice, its MAS on hand-built cases, the prior's
lgamma form against scipy; and a written filelist read back through the reference's own TTSDataset."""
import ctypes as C
import math
import os
import re
import sys

import numpy as np
import pytest
import scipy.stats
import torch
import torch.nn.functional as F

from conftest import GOLDEN, REPO
from fastspeech2_b200 import _lib
from fastspeech2_b200 import aligner as A
from oracle import aligner_oracle as O
from oracle import ref_import

NEW = ("fs2_align_workspace_bytes", "fs2_align_logprob", "fs2_align_logprob_backward", "fs2_align_forward_sum", "fs2_align_mas",
       "fs2_align_bin_loss", "fs2_align_mask_rows")
LINE = "Some text, here.|-2 4 7 14|6 3 7|HH AH0 pau|LJ001-0001.wav"


def test_abi_symbols_are_exported_and_declared():
    lib = _lib.load()
    header = open(os.path.join(REPO, "include", "fs2_b200.h")).read()
    for name in NEW:
        assert hasattr(lib, name) and name in _lib.SIGNATURES, name
        assert re.search(r"\b%s\(" % name, header), name
    for bit in ("FS2_ALIGN_BAD_LENGTH 1", "FS2_ALIGN_INFEASIBLE 2", "FS2_ALIGN_NONFINITE 4", "FS2_ALIGN_DIM 80", "FS2_ALIGN_MAX_T 1024"):
        assert "#define " + bit in header


def test_filelist_round_trip(tmp_path):
    ln = A.parse_line(LINE)
    assert (ln.text, ln.boundaries, ln.durations, ln.phonemes, ln.wav, ln.id) == \
        ("Some text, here.", [-2, 4, 7, 14], [6, 3, 7], ["HH", "AH0", "pau"], "LJ001-0001.wav", "LJ001-0001")
    out = A.format_line(ln, [2, 5, 1])
    assert out == "Some text, here.|0 2 7 8|2 5 1|HH AH0 pau|LJ001-0001.wav"
    back = A.parse_line(out)
    assert back.durations == [2, 5, 1] and back.boundaries == [0, 2, 7, 8] and back.phonemes == ln.phonemes
    bare = A.parse_line("text||| AA B  |x.wav\n")          # fields 1 and 2 empty
    assert bare.boundaries is None and bare.durations is None and bare.phonemes == ["AA", "B"]
    p = tmp_path / "f.txt"
    p.write_text(LINE + "\n\n" + out + "\n")
    assert [x.durations for x in A.read_filelist(str(p))] == [[6, 3, 7], [2, 5, 1]]


@pytest.mark.parametrize("line, match", [
    ("a|b|c|d", "expected 5 '|'-separated fields, found 4"),
    ("t|1 x|1|AA|w.wav", "field 2 must hold integers"),
    ("t||1 2|AA|w.wav", "2 durations for 1 phonemes"),
    ("t|||  |w.wav", "no phonemes"),
    ("t|||AA| ", "no wav name"),
])
def test_filelist_errors_name_the_line(line, match):
    with pytest.raises(ValueError, match="^list.txt:3: " + match):
        A.parse_line(line, "list.txt:3")


def test_symbol_table_is_the_sorted_token_set():
    lines = [A.parse_line("t|||B AA pau|a.wav"), A.parse_line("t|||AA sil B|b.wav")]
    sym = A.build_symbols(lines)
    assert sym == ["<pad>", "AA", "B", "pau", "sil"]
    assert A.encode(lines[0], sym).tolist() == [2, 1, 3]
    with pytest.raises(ValueError, match=r"phonemes \['ZH'\] are not in the aligner's symbol table"):
        A.encode(A.parse_line("t|||AA ZH|c.wav"), sym)
    with pytest.raises(ValueError, match="not in the aligner's symbol table"):
        A.encode(A.parse_line("t|||<pad>|c.wav"), sym)


def test_workspace_formula():
    a256 = lambda v: (v + 255) // 256 * 256     # noqa: E731
    for B, L, T in ((1, 1, 1), (32, 800, 100), (3, 17, 1024)):
        assert A.workspace_bytes(B, L, T) == a256(4 * B) + a256(4 * B * L) + 4 * B * L * (2 * T + 1)


@pytest.mark.parametrize("B, L, T, match", [(0, 1, 1, r"B \(0\)"), (65536, 1, 1, r"B \(65536\)"), (1, 0, 1, r"L \(0\)"),
                                            (1, 1, 0, r"T \(0\)"), (1, 1, 1025, r"T \(1025\) must lie in \[1, 1024\]")])
def test_c_refusals_name_their_argument(B, L, T, match):
    n = C.c_size_t()
    assert _lib.load().fs2_align_workspace_bytes(B, L, T, C.byref(n)) == -1
    assert re.search(match, _lib.load().fs2_last_error().decode())


def test_c_entries_refuse_null_arguments_and_bad_workspace_without_a_gpu():
    lib = _lib.load()
    p = C.c_void_p(256)
    calls = {
        "fs2_align_logprob": lambda q: lib.fs2_align_logprob(q, p, p, p, 1, 4, 2, p, p, p, 1 << 20, None),
        "fs2_align_logprob_backward": lambda q: lib.fs2_align_logprob_backward(q, p, p, p, 1, 4, 2, p, p, p, p, p, 1 << 20, None),
        "fs2_align_forward_sum": lambda q: lib.fs2_align_forward_sum(q, p, p, 1, 4, 2, None, p, None, p, p, 1 << 20, None),
        "fs2_align_mas": lambda q: lib.fs2_align_mas(q, p, p, 1, 4, 2, p, p, p, p, 1 << 20, None),
        "fs2_align_bin_loss": lambda q: lib.fs2_align_bin_loss(q, p, p, p, 1, 4, 2, None, p, None, p, p, 1 << 20, None),
    }
    for name, call in calls.items():
        assert call(None) == -1
        assert lib.fs2_last_error().decode() == f"{name}: null argument"
    assert lib.fs2_align_mas(p, p, p, 1, 4, 2, p, p, p, p, 16, None) == -4            # short workspace
    assert "fs2_align_mas: workspace too small" in lib.fs2_last_error().decode()
    assert lib.fs2_align_forward_sum(p, p, p, 1, 4, 2, None, p, None, p, C.c_void_p(8), 1 << 20, None) == -1
    assert "256-byte aligned" in lib.fs2_last_error().decode()
    assert lib.fs2_align_mask_rows(None, p, 1, 1, 1, p, None) == -1
    assert lib.fs2_align_mask_rows(p, p, 1, 0, 1, p, None) == -1
    assert lib.fs2_align_workspace_bytes(1, 1, 1, None) == -1


def test_module_checks_its_inputs():
    with pytest.raises(ValueError, match="n_symbols must be an integer >= 2"):
        A.Aligner(1)
    xs, il, mel, ol = torch.ones(2, 3, dtype=torch.int64), torch.tensor([3, 2]), torch.zeros(2, 5, 80), torch.tensor([5, 4])
    for args, match in [((xs.float(), il, mel, ol), r"xs must be a \[B, T\] integer tensor"),
                        ((xs, il, mel.double(), ol), r"mels must be a \[B, L, 80\] float32 tensor"),
                        ((xs, il, mel[:1], ol), "mels has 1 utterances, xs 2"),
                        ((torch.ones(1, 1025, dtype=torch.int64), il[:1], mel[:1], ol[:1]), "T = 1025 phonemes exceeds"),
                        ((xs, il[:1], mel, ol), r"ilens must be a \[B=2\] integer tensor"),
                        ((xs, il, mel, ol.float()), r"olens must be a \[B=2\] integer tensor"),
                        ((xs, il, mel, ol), "must be CUDA tensors")]:
        with pytest.raises(ValueError, match=match):
            A.Aligner._inputs(*args)


def test_state_dict_layout():
    sd = A.Aligner(12).state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == {
        "embed.weight": (12, 256), "key_conv1.weight": (512, 256, 3), "key_conv1.bias": (512,), "key_conv2.weight": (80, 512, 1),
        "key_conv2.bias": (80,), "query_conv1.weight": (160, 80, 3), "query_conv1.bias": (160,), "query_conv2.weight": (80, 160, 1),
        "query_conv2.bias": (80,), "query_conv3.weight": (80, 80, 1), "query_conv3.bias": (80,)}
    assert not sd["embed.weight"][0].any()


def test_kernels_do_not_spill():
    path = os.path.join(REPO, "fastspeech2_b200", "build", "aligner.ptxas.txt")
    if not os.path.exists(path):
        pytest.skip("no ptxas reports (library built elsewhere)")
    text = open(path).read()
    for kernel in ("al_check_kernel", "al_logprob_kernel", "al_logprob_dq_kernel", "al_logprob_dk_kernel", "al_forward_sum_kernel",
                   "al_mas_kernel", "al_bin_loss_kernel", "al_mask_rows_kernel"):
        props = re.findall(r"Function properties for \S*%s\S*\n(.*)" % kernel, text)
        assert props, kernel
        for line in props:
            assert "0 bytes spill stores, 0 bytes spill loads" in line, (kernel, line)


# ---- the oracle ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N, M", [(1, 1), (1, 6), (2, 2), (3, 7), (5, 5), (4, 11)])
def test_forward_sum_is_ctc_on_the_blank_augmented_lattice(N, M):
    lp = torch.from_numpy(np.random.default_rng(N * 31 + M).standard_normal((1, M, N)) * 2)
    got = float(O.forward_sum(lp, [N], [M])[0])
    ls = torch.log_softmax(F.pad(lp[0], (1, 0), value=-1.0), 1).numpy()
    assert got == pytest.approx(O.ctc_direct(ls) / N, rel=1e-12)


def test_forward_sum_of_an_infeasible_utterance_is_zero():
    lp = torch.zeros(2, 3, 4, dtype=torch.float64, requires_grad=True)
    out = O.forward_sum(lp, [4, 2], [3, 3])
    assert float(out[0]) == 0.0 and float(out[1]) > 0
    out[0].backward()
    assert not lp.grad.any()


def test_prior_lgamma_form_matches_scipy():
    """The kernel's float64 form: log pmf = lgamma terms of C(N, t) B(t + a, N - t + b) / B(a, b)."""
    for N, M in ((1, 1), (1, 5), (7, 7), (13, 90), (100, 800)):
        ref = O.prior(N, M)
        for l in range(0, M, max(1, M // 7)):
            a, b = l + 1.0, float(M - l)
            rowc = math.lgamma(N + 1) - math.lgamma(N + a + b) - math.lgamma(a) - math.lgamma(b) + math.lgamma(a + b)
            got = np.array([math.exp(rowc - math.lgamma(t + 1) - math.lgamma(N - t + 1) + math.lgamma(t + a) + math.lgamma(N - t + b))
                            for t in range(N)])
            np.testing.assert_allclose(got, ref[l], rtol=1e-9, atol=1e-300)
    assert O.prior(4, 1)[0].tolist() == pytest.approx(scipy.stats.betabinom(4, 1, 1).pmf(range(4)).tolist())


def _durs(path, N):
    return np.bincount(path, minlength=N)


def test_mas_ties_go_to_the_earlier_phoneme():
    # every entry equal: each step ties, and t - 1 wins, so the path stays on phoneme 0 until it must move
    p = O.mas_width1(np.zeros((6, 3), np.float32))
    assert p.tolist() == [0, 0, 0, 0, 1, 2]
    # frames 2 and 3 each tie between staying and advancing (v = -1 / -1, then -3 / -3): both go to the earlier
    # phoneme, giving [0, 0, 1, 2] where the later one would give [0, 1, 2, 2]
    ls = np.array([[0, -9, -9], [-1, -1, -9], [-9, -2, -2], [-9, -9, 0]], np.float32)
    assert O.mas_width1(ls).tolist() == [0, 0, 1, 2]


def test_mas_edges():
    rng = np.random.default_rng(3)
    ls = np.log(rng.dirichlet(np.ones(5), size=5)).astype(np.float32)
    assert O.mas_width1(ls).tolist() == [0, 1, 2, 3, 4]                     # L == T: one frame each
    assert O.mas_width1(ls[:, :1]).tolist() == [0] * 5                       # one phoneme
    assert O.mas_width1(ls[:1, :1]).tolist() == [0]                          # one frame
    big = np.log(rng.dirichlet(np.ones(7), size=40)).astype(np.float32)
    d = _durs(O.mas_width1(big), 7)
    assert d.min() >= 1 and d.sum() == 40


def test_mas_follows_a_clear_alignment():
    truth = np.array([3, 1, 5, 2])
    path = np.repeat(np.arange(4), truth)
    ls = np.full((truth.sum(), 4), -20.0, np.float32)
    ls[np.arange(truth.sum()), path] = -0.01
    assert _durs(O.mas_width1(O.log_soft32(ls)), 4).tolist() == truth.tolist()
    dur, pth = O.mas(np.pad(ls, ((0, 2), (0, 1)))[None], [4], [truth.sum()])
    assert dur[0].tolist() == truth.tolist() + [0] and pth[0].tolist() == path.tolist() + [-1, -1]


def test_bin_loss_oracle():
    lp = torch.log(torch.tensor([[[0.5, 0.5], [0.1, 0.9], [0.0, 0.0]]], dtype=torch.float64))
    got = float(O.bin_loss(lp, [[0, 1, -1]], [2], [2])[0])
    assert got == pytest.approx(-(math.log(0.5) + math.log(0.9)) / 2)


# ---- the reference's loader reads what extract writes -------------------------------------------------------------------
def test_written_filelist_reads_back_through_the_reference_loader(tmp_path):
    if not ref_import.available():
        pytest.skip("no reference staged in oracle/_ref (oracle/stage_ref.py)")
    z = np.load(os.path.join(GOLDEN, "align_filelist.npz"))
    rng = np.random.default_rng(0)
    root = tmp_path / "data"
    for d in ("mels", "energy", "pitch"):
        (root / d).mkdir(parents=True)
    lines, want = [], []
    for i in range(6):
        ln = A.parse_line(f"t|||{z['phonemes'][i]}|{z['wavs'][i]}")
        N = len(ln.phonemes)
        d = rng.integers(1, 9, N)
        L = int(d.sum())
        np.save(root / "mels" / f"{ln.id}.npy", rng.standard_normal((80, L)).astype(np.float32))
        np.save(root / "energy" / f"{ln.id}.npy", rng.random(L).astype(np.float32) + 0.1)
        np.save(root / "pitch" / f"{ln.id}.npy", rng.random(L) * 200 + 80)
        lines.append(A.format_line(ln, d))
        want.append((d, L))
    fl = tmp_path / "aligned.txt"
    fl.write_text("\n".join(lines) + "\n")
    exec(ref_import.STUB_SNIPPET, {})
    sys.path.insert(0, ref_import.REF_DIR)
    try:
        from dataset.dataloader import TTSDataset          # the reference's loader (dataset/dataloader.py:47-74)
        ds = TTSDataset(str(root) + "/", str(fl), True, ["english_cleaners"], False)
        for i, (d, L) in enumerate(want):
            x, mel, _, mel_len, dur, _, _ = ds[i]
            assert mel_len == L == int(dur.sum()) and mel.shape == (L, 80)
            assert dur.tolist() == d.tolist()                # its last-duration correction changed nothing
            assert len(x) == len(d)
    finally:
        sys.path.remove(ref_import.REF_DIR)
