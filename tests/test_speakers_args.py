"""Multi-speaker FastSpeech2 (DESIGN.md section 25) without a GPU: the speaker oracle against the unmodified reference
(tests/golden/speakers.npz), the checkpoint layout, the argument errors that need no device, the six-field filelists,
speaker maps and the collation of speaker ids."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from fastspeech2_b200 import FeedForwardTransformer
from fastspeech2_b200 import aligner as A
from fastspeech2_b200 import data as D
from fastspeech2_b200 import speakers as S
from fastspeech2_b200.hparams import load_hp
from oracle import speaker_oracle as SO
import _speakers_golden as SG

T = torch.from_numpy


def hp_with(n):
    hp = load_hp()
    hp["model"]["n_speakers"] = n
    return hp


def close(a, b, tol=1e-6):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.max(np.abs(a - b)) <= tol, float(np.max(np.abs(a - b)))


# ---- the oracle against the reference -------------------------------------------------------------------------------------
def test_speaker_oracle_matches_reference(golden, weights):
    g = golden("speakers")
    tab, spk = T(g["table"]), T(g["speakers"])
    torch.set_num_threads(1)
    with torch.no_grad():
        b, a, d, e, p = SO.forward_path(weights, tab, spk, T(g["xs"]), T(g["ilens"]), T(g["olens"]), T(g["ds"]).clone(),
                                        T(g["es"]), T(g["ps"]), False)
        close(d, g["tf_d_outs"]); close(e, g["tf_e_outs"]); close(p, g["tf_p_outs"])
        mels, means = SG.mel_checks(g, "tf", b, a, T(g["olens"]))
        for _, got, want in mels + means:
            close(got, want)
        b, a, d, eh, ph = SO.forward_path(weights, tab, spk, T(g["xs"]), T(g["ilens"]), is_inference=True)
    assert torch.equal(d, T(g["inf_d_outs"])) and a.shape[1] == int(g["inf_frames"])
    assert torch.equal(eh.argmax(-1), T(g["inf_e_ids"]).long()) and torch.equal(ph.argmax(-1), T(g["inf_p_ids"]).long())
    mels, means = SG.mel_checks(g, "inf", b, a, d.sum(1))
    for _, got, want in mels + means:
        close(got, want)


def test_golden_batch_and_gradient_samples_are_regenerated(golden):
    """ys comes from make_batch and the gradient indices from sample_indices: both must match what was stored."""
    g = golden("speakers")
    SG.batch(g)
    numels = {k: v.numel() for k, v in FeedForwardTransformer(68, 80, load_hp()).named_parameters()}
    samples = SG.grad_samples(g, numels)
    assert set(samples) == set(numels) - set(json.loads(str(g["no_grad"])))


def test_golden_speakers_matter_and_one_is_absent(golden):
    g = golden("speakers")
    assert set(g["speakers"].tolist()) == {0, 1, 2, 3} and int(g["n_speakers"]) == 5
    assert np.all(g["grad/speaker_embed.weight"][4] == 0) and np.abs(g["grad/speaker_embed.weight"][:4]).min(axis=1).max() > 0


# ---- checkpoint layout ----------------------------------------------------------------------------------------------------
def test_state_dict_keys():
    ref = json.load(open(os.path.join(GOLDEN, "state_dict_keys.json")))
    keys = [[k, list(v.shape), str(v.dtype)] for k, v in FeedForwardTransformer(68, 80, load_hp()).state_dict().items()]
    assert keys == ref
    assert [[k, list(v.shape), str(v.dtype)] for k, v in FeedForwardTransformer(68, 80, hp_with(0)).state_dict().items()] == ref
    m = FeedForwardTransformer(68, 80, hp_with(7))
    keys = [[k, list(v.shape), str(v.dtype)] for k, v in m.state_dict().items()]
    assert keys == ref + [["speaker_embed.weight", [7, 256], "torch.float32"]]
    assert m.speaker_embed.padding_idx is None


def test_other_parameters_initialise_as_in_the_single_speaker_model():
    torch.manual_seed(3)
    a = FeedForwardTransformer(68, 80, load_hp()).state_dict()
    torch.manual_seed(3)
    b = FeedForwardTransformer(68, 80, hp_with(4)).state_dict()
    assert all(torch.equal(a[k], b[k]) for k in a)
    assert abs(float(b["speaker_embed.weight"].std()) - 1.0) < 0.2     # nn.Embedding's N(0, 1)


def test_from_checkpoint_reads_the_speaker_count(tmp_path, weights):
    from fastspeech2_b200.hparams import load_hp_str
    sd = dict(weights)
    sd["speaker_embed.weight"] = torch.zeros(6, 256)
    with open(os.path.join(os.path.dirname(GOLDEN), "..", "fastspeech2_b200", "configs", "default.yaml")) as fh:
        hp_str = fh.read()                                  # written before the key existed
    assert "n_speakers" not in load_hp_str(hp_str)["model"]
    m = FeedForwardTransformer.from_checkpoint({"model": sd, "hp_str": hp_str})
    assert m.n_speakers == 6 and tuple(m.speaker_embed.weight.shape) == (6, 256)
    with pytest.raises(ValueError, match="n_speakers = 3 but the checkpoint's speaker table has 6 rows"):
        FeedForwardTransformer.from_checkpoint({"model": sd, "hp_str": hp_str}, hp=hp_with(3))
    with pytest.raises(ValueError, match="n_speakers = 3 but the checkpoint's speaker table has 0 rows"):
        FeedForwardTransformer.from_checkpoint({"model": dict(weights), "hp_str": hp_str}, hp=hp_with(3))
    assert FeedForwardTransformer.from_checkpoint({"model": dict(weights), "hp_str": hp_str}).n_speakers == 0


# ---- argument errors that need no device -----------------------------------------------------------------------------------
@pytest.mark.parametrize("n, speakers, match", [
    (4, None, "the model has 4 speakers: pass the speaker ids"),
    (0, torch.zeros(2, dtype=torch.int64), "the model has no speaker table"),
    (4, torch.tensor([0, 4]), r"1 id\(s\) outside \[0, n_speakers=4\)"),
    (4, torch.tensor([-1, 0]), r"1 id\(s\) outside \[0, n_speakers=4\)"),
    (4, torch.zeros(3, dtype=torch.int64), r"speakers must be \[B=2\]"),
    (4, torch.zeros(2, 1, dtype=torch.int64), r"speakers must be \[B=2\]"),
    (4, torch.zeros(2, dtype=torch.int32), "speakers must be an int64 tensor"),
    (4, [0, 1], "speakers must be an int64 tensor"),
])
def test_speaker_errors(n, speakers, match):
    m = FeedForwardTransformer(68, 80, hp_with(n)).eval()
    xs, il = torch.ones(2, 5, dtype=torch.int64), torch.tensor([5, 3])
    with pytest.raises(ValueError, match=match):
        m.synthesize(xs, il, speakers=speakers)
    with pytest.raises(ValueError, match=match):
        m._forward(xs, il, is_inference=True, speakers=speakers)


def test_inference_speaker_errors():
    m = FeedForwardTransformer(68, 80, hp_with(3)).eval()
    x = torch.ones(5, dtype=torch.int64)
    with pytest.raises(ValueError, match="pass the speaker ids"):
        m.inference(x)
    with pytest.raises(ValueError, match="outside"):
        m.inference(x, 3)
    with pytest.raises(ValueError, match="an int or a 0-d"):
        m.inference(x, torch.tensor([1]))
    with pytest.raises(ValueError, match="an int or a 0-d"):
        m.inference(x, 1.0)
    with pytest.raises(ValueError, match="outside"):
        m.inference_controlled(x, speed=1.2, speaker=-1)
    with pytest.raises(ValueError, match="no speaker table"):
        FeedForwardTransformer(68, 80, load_hp()).eval().inference(x, 0)


def test_bad_hp_speaker_count():
    with pytest.raises(ValueError, match="n_speakers must be an int >= 0"):
        FeedForwardTransformer(68, 80, hp_with(-2))
    with pytest.raises(ValueError, match="n_speakers must be an int >= 0"):
        FeedForwardTransformer(68, 80, hp_with("4"))


# ---- filelists and speaker maps --------------------------------------------------------------------------------------------
LINE5 = "Hello there.|0 2 7 8|2 5 1|HH AH L|p225_003.wav"


def test_five_and_six_field_lines_round_trip():
    a = A.parse_line(LINE5)
    assert a.speaker is None and A.format_line(a, a.durations) == LINE5
    b = A.parse_line(LINE5 + "|p225\n")
    assert b.speaker == "p225" and b.wav == "p225_003.wav" and b.durations == [2, 5, 1]
    assert A.format_line(b, b.durations) == LINE5 + "|p225"
    assert A.format_line(b, [1, 1, 6]) == "Hello there.|0 1 2 8|1 1 6|HH AH L|p225_003.wav|p225"


@pytest.mark.parametrize("line, match", [
    (LINE5 + "|p225|x", "expected 5 '|'-separated fields, found 7"),
    (LINE5 + "| ", "empty speaker field"),
])
def test_bad_speaker_fields(line, match):
    with pytest.raises(ValueError, match="^f:1: " + match):
        A.parse_line(line, "f:1")


def test_extract_keeps_the_speaker_field(tmp_path, monkeypatch):
    """`aligner extract` writes each line through format_line: the speaker field is carried through."""
    lines = [A.parse_line(LINE5 + "|p225"), A.parse_line("t|||AA B|19_198_000000_000000.wav")]
    monkeypatch.setattr(A, "read_filelist", lambda path: lines)
    monkeypatch.setattr(A, "load", lambda path: (None, ["<pad>", "AA", "AH", "B", "HH", "L"], 1))

    class FakeCorpus:
        def __init__(self, lines, symbols, data_dir, log=None):
            self.lines = lines
    monkeypatch.setattr(A, "Corpus", FakeCorpus)
    monkeypatch.setattr(A, "extract", lambda model, corpus, batch=32: [np.array([3, 3, 2]), np.array([1, 4])])
    cfg = tmp_path / "c.yaml"
    cfg.write_text("data:\n  data_dir: " + str(tmp_path) + "\n")
    out = tmp_path / "out.txt"
    A.main(["extract", "-c", str(cfg), "--filelist", "x", "-p", "ck.pt", "--out", str(out)])
    got = out.read_text().splitlines()
    assert got[0] == "Hello there.|0 3 6 8|3 3 2|HH AH L|p225_003.wav|p225"
    assert got[1] == "t|0 1 5|1 4|AA B|19_198_000000_000000.wav"


def test_speaker_names_and_maps(tmp_path):
    assert S.speaker_from_wav("p225_003.wav") == "p225"
    assert S.speaker_from_wav("19_198_000000_000000.wav") == "19"
    assert S.speaker_from_wav("wavs/p226_001") == "p226"
    lines = [A.parse_line(f"t|||AA|{w}") for w in ("p226_1.wav", "p225_2.wav", "p226_3.wav", "p300_1.wav")]
    m1, m2 = S.build_map(lines), S.build_map(lines[::-1])
    assert m1 == m2 == {"p225": 0, "p226": 1, "p300": 2} and list(m1) == ["p225", "p226", "p300"]
    S.save_map(str(tmp_path / "m.json"), m1)
    assert S.load_map(str(tmp_path / "m.json")) == m1
    (tmp_path / "bad.json").write_text('{"a": 0, "b": 2}')
    with pytest.raises(ValueError, match="not a speaker map"):
        S.load_map(str(tmp_path / "bad.json"))


def test_speakers_tag_round_trips(tmp_path):
    src = tmp_path / "in.txt"
    src.write_text(LINE5 + "\n\nt||1 1|AA B|19_198_000000_000000.wav\nt|||AA|p226_9.wav|custom\n")
    dst = tmp_path / "out.txt"
    S.main(["tag", str(src), str(dst), "--map", str(tmp_path / "spk.json")])
    got = dst.read_text().splitlines()
    assert got == [LINE5 + "|p225", "t||1 1|AA B|19_198_000000_000000.wav|19", "t|||AA|p226_9.wav|custom"]
    assert S.load_map(str(tmp_path / "spk.json")) == {"19": 0, "custom": 1, "p225": 2}
    assert [ln.speaker for ln in A.read_filelist(str(dst))] == ["p225", "19", "custom"]
    S.tag(str(dst), str(tmp_path / "again.txt"))            # already tagged: unchanged, map beside the output
    assert (tmp_path / "again.txt").read_text() == dst.read_text()
    assert S.load_map(str(tmp_path / "speakers.json")) == {"19": 0, "custom": 1, "p225": 2}


# ---- collation -------------------------------------------------------------------------------------------------------------
def _items(with_speakers):
    g = np.random.RandomState(5)
    out = []
    for i, (Tn, L) in enumerate([(7, 31), (12, 50), (3, 9)]):
        it = (g.randint(1, 68, size=Tn), g.randn(L, 80).astype(np.float32), f"u{i}", L, g.randint(1, 6, size=Tn),
              g.rand(L).astype(np.float32), g.rand(L).astype(np.float32))
        out.append(it + ((4, 0, 4)[i],) if with_speakers else it)
    return out


def _equal(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert torch.equal(x, y) if torch.is_tensor(x) else x == y


def test_collation_with_and_without_speakers():
    plain, tagged = _items(False), _items(True)
    base = D.collate_tts(plain)
    assert len(base) == 9
    out = D.collate_tts(tagged)
    assert len(out) == 10
    _equal(out[:9], base)
    assert out[9].dtype == torch.int64 and out[9].tolist() == [4, 0, 4]
    pc = D.PinnedCollator(4, 16, 64, pin=False)
    p9 = pc(plain)
    assert len(p9) == 9
    _equal(p9, base)
    p10 = pc(tagged)
    assert len(p10) == 10
    _equal(p10[:9], base)
    assert p10[9].tolist() == [4, 0, 4]
    with pytest.raises(ValueError, match="all 8"):
        D.collate_tts(plain[:1] + tagged[1:])


def test_filelist_dataset_reads_a_preprocess_tree(tmp_path):
    from fastspeech2_b200.preprocess import remove_outlier
    for kind in ("mels", "energy", "pitch"):
        (tmp_path / kind).mkdir()
    g = np.random.RandomState(0)
    mel = g.randn(80, 12).astype(np.float32)
    e = g.rand(12).astype(np.float32) * 50
    e[3] = 1e4                                            # an outlier
    p = g.rand(12).astype(np.float32) * 300
    np.save(tmp_path / "mels" / "p225_003.npy", mel)
    np.save(tmp_path / "energy" / "p225_003.npy", e)
    np.save(tmp_path / "pitch" / "p225_003.npy", p)
    fl = tmp_path / "f.txt"
    fl.write_text("t||2 5 1|HH AH L|p225_003.wav|p225\n")
    sym = A.build_symbols(A.read_filelist(str(fl)))
    ds = D.FilelistDataset(str(fl), str(tmp_path), sym, {"p225": 3, "p226": 0})
    x, m, uid, L, d, ee, pp, s = ds[0]
    assert x.tolist() == [2, 1, 3] and uid == "p225_003" and L == 12 and s == 3
    assert np.array_equal(m, mel.T) and d.tolist() == [2, 5, 5]             # last duration stretched to the 12 frames
    assert np.array_equal(ee, remove_outlier(e.copy())) and np.array_equal(pp, remove_outlier(p.copy()))
    assert len(D.FilelistDataset(str(fl), str(tmp_path), sym)[0]) == 7
    assert ds.mel_lengths() == [12]
    with pytest.raises(ValueError, match="not in the speaker map"):
        D.FilelistDataset(str(fl), str(tmp_path), sym, {"p226": 0})
