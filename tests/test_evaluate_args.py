"""Objective evaluation without a device: the argument checks of mcd_dtw / path_prosody, the C entries' size checks and
workspace formula, and the evaluate command's id pairing, missing-file errors and budgeted batching on tiny `.npy` trees
(the device entry replaced by the float64 oracle)."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib
from fastspeech2_b200 import evaluate as EV
from oracle import eval_oracle as E


def _xy(B=2, Lx=5, Ly=6, M=8):
    return (torch.zeros(B, Lx, M), torch.full((B,), Lx), torch.zeros(B, Ly, M), torch.full((B,), Ly))


@pytest.mark.parametrize("change, match", [
    (lambda a: {"x": a["x"][0]}, "x must be a non-empty"),
    (lambda a: {"x": a["x"][:, :0]}, "x must be a non-empty"),
    (lambda a: {"y": a["y"].double()}, "y must be float32"),
    (lambda a: {"x": a["x"].half()}, "x must be float32"),
    (lambda a: {"y": a["y"][:1]}, "y has 1 utterances, x has 2"),
    (lambda a: {"y": a["y"][:, :, :7]}, "y has n_mels=7, x has n_mels=8"),
    (lambda a: {"xlens": a["xlens"][:1]}, r"xlens must be a \[B=2\] tensor"),
    (lambda a: {"ylens": a["ylens"].float()}, "ylens must be an integer tensor"),
    (lambda a: {"xlens": a["xlens"].bool()}, "xlens must be an integer tensor"),
    (lambda a: {"n_cep": 0}, r"n_cep must be an integer in \[1, n_mels - 1 = 7\]"),
    (lambda a: {"n_cep": 8}, r"n_cep must be an integer in \[1, n_mels - 1 = 7\]"),
    (lambda a: {"n_cep": 2.0}, "n_cep must be an integer"),
    (lambda a: {"n_cep": True}, "n_cep must be an integer"),
    (lambda a: {}, "x, xlens, y and ylens must be CUDA tensors"),
])
def test_mcd_dtw_argument_checks(change, match):
    x, xl, y, yl = _xy()
    a = {"x": x, "xlens": xl, "y": y, "ylens": yl, "n_cep": 7}
    a.update(change(a))
    with pytest.raises(ValueError, match=match):
        EV.mcd_dtw(a["x"], a["xlens"], a["y"], a["ylens"], n_cep=a["n_cep"])


def _prosody_args(B=2):
    return {"path": torch.zeros(B, 10, 2, dtype=torch.int32), "plen": torch.full((B,), 5), "f0x": torch.zeros(B, 5, dtype=torch.float64),
            "f0x_lens": torch.full((B,), 5), "f0y": torch.zeros(B, 6, dtype=torch.float64), "f0y_lens": torch.full((B,), 6),
            "ex": torch.zeros(B, 5), "ey": torch.zeros(B, 6)}


@pytest.mark.parametrize("change, match", [
    (lambda a: {"path": a["path"][:, :, 0]}, r"path must be a non-empty \[B, P_max, 2\]"),
    (lambda a: {"path": a["path"].long()}, "path must be int32"),
    (lambda a: {"plen": a["plen"][:1]}, r"plen must be a \[B=2\] tensor"),
    (lambda a: {"plen": a["plen"].double()}, "plen must be an integer tensor"),
    (lambda a: {"f0x": a["f0x"].float()}, "f0x must be torch.float64"),
    (lambda a: {"f0y": a["f0y"][:1]}, r"f0y must be a non-empty \[B=2, L\]"),
    (lambda a: {"ex": a["ex"].double()}, "ex must be torch.float32"),
    (lambda a: {"ey": a["ey"][:, :0]}, r"ey must be a non-empty \[B=2, L\]"),
    (lambda a: {"f0x_lens": a["f0x_lens"].float()}, "f0x_lens must be an integer tensor"),
    (lambda a: {"f0y_lens": a["f0y_lens"][:1]}, r"f0y_lens must be a \[B=2\] tensor"),
    (lambda a: {}, "must be CUDA tensors"),
])
def test_path_prosody_argument_checks(change, match):
    a = _prosody_args()
    a.update(change(a))
    with pytest.raises(ValueError, match=match):
        EV.path_prosody(**a)


def _ws(*args):
    n = C.c_size_t()
    return _lib.load().fs2_dtw_workspace_bytes(*args, C.byref(n)), n.value


def test_workspace_formula_and_no_product_without_a_path():
    a256 = lambda v: (v + 255) // 256 * 256     # noqa: E731
    B, M, K = 4, 80, 24
    for Lx, Ly in ((300, 500), (1024, 5000), (1025, 5000), (4100, 4200)):
        W = min(Lx, Ly)
        base = a256(8 * B * Lx * K) + a256(8 * B * Ly * K) + ((a256(8 * B * 3 * W) + a256(4 * B * 3 * W)) if W > 1024 else 0)
        assert _ws(B, Lx, Ly, M, K, 0) == (0, a256(base) + 256)
        assert _ws(B, Lx, Ly, M, K, 1) == (0, a256(a256(base) + B * (Lx + Ly - 1) * W) + 256)
    for L in (400, 1100):                    # both sides of the shared-memory limit
        small, big = _ws(B, L, L, M, K, 0)[1], _ws(B, 2 * L, 2 * L, M, K, 0)[1]
        assert big <= 2 * small + 1024       # doubling both lengths doubles it, it does not quadruple it
        assert _ws(B, 2 * L, 2 * L, M, K, 1)[1] > 3 * _ws(B, L, L, M, K, 1)[1]


@pytest.mark.parametrize("args, match", [
    ((0, 5, 5, 80, 24, 0), "B"),
    ((1, 0, 5, 80, 24, 0), "Lx_max and Ly_max"),
    ((1, 5, 5, 1, 1, 0), "n_mels"),
    ((1, 5, 5, 80, 0, 0), "n_cep"),
    ((1, 5, 5, 80, 80, 0), r"n_cep \(80\) must lie in \[1, n_mels - 1 = 79\]"),
])
def test_c_size_checks(args, match):
    rc, _ = _ws(*args)
    assert rc == -1
    assert re.search(match, _lib.load().fs2_last_error().decode())


def test_c_entries_refuse_null_arguments_without_a_gpu():
    lib = _lib.load()
    assert lib.fs2_mcd_dtw(None, None, 5, None, None, 5, 1, 80, None, 24, 1.0, None, None, None, None, None, None, 0, None) == -1
    assert "null argument" in lib.fs2_last_error().decode()
    assert lib.fs2_path_prosody(None, None, 1, 5, None, None, 5, None, None, 5, None, 5, None, 5, None, None, None, None) == -1


# ---- the command ----------------------------------------------------------------------------------------------------

def _tree(root, ids, lens, seed, M=8, pitch=True, energy=True):
    rng = np.random.default_rng(seed)
    for d in ("mels",) + (("pitch",) if pitch else ()) + (("energy",) if energy else ()):
        os.makedirs(os.path.join(root, d), exist_ok=True)
    for uid, T in zip(ids, lens):
        np.save(os.path.join(root, "mels", uid + ".npy"), rng.uniform(-11, 1, (M, T)).astype(np.float32))
        if pitch:
            f0 = np.where(rng.random(T - 1) < 0.3, 0.0, rng.uniform(80, 250, T - 1))
            np.save(os.path.join(root, "pitch", uid + ".npy"), f0)
        if energy:
            np.save(os.path.join(root, "energy", uid + ".npy"), rng.uniform(0, 5, T).astype(np.float32))


oracle_score = E.backend


def test_command_pairs_ids_and_writes_rows(tmp_path):
    ids = ["b", "a", "c"]
    _tree(tmp_path / "ref", ids, [7, 9, 4], 0)
    _tree(tmp_path / "syn", ids, [8, 9, 3], 1)
    out = EV.run(str(tmp_path / "ref"), str(tmp_path / "syn"), n_cep=5, csv_path=str(tmp_path / "rows.csv"), score=oracle_score(5))
    assert out["utterances"] == 3 and out["n_cep"] == 5
    rows = open(tmp_path / "rows.csv").read().splitlines()
    assert rows[0].startswith("id,lx,ly,mcd_db,cost,path_len") and [r.split(",")[:3] for r in rows[1:]] == \
        [["a", "9", "9"], ["b", "8", "7"], ["c", "3", "4"]]
    assert out["length_ratio"] == np.mean([9 / 9, 8 / 7, 3 / 4])
    assert all(out[k] is not None for k in ("mcd_db", "f0_rmse_cents", "vuv_error", "gpe", "ffe", "energy_rmse"))
    json.dumps(out)


def test_command_against_itself_is_zero(tmp_path):
    _tree(tmp_path / "ref", ["u1", "u2"], [6, 11], 0)
    out = EV.run(str(tmp_path / "ref"), str(tmp_path / "ref"), n_cep=7, score=oracle_score(7))
    for k in ("mcd_db", "f0_rmse_cents", "vuv_error", "gpe", "ffe", "energy_rmse"):
        assert out[k] == 0.0, k
    assert out["length_ratio"] == 1.0


def test_command_ids_file_and_missing_reference(tmp_path):
    _tree(tmp_path / "ref", ["a"], [5], 0)
    _tree(tmp_path / "syn", ["a", "b"], [5, 6], 1)
    (tmp_path / "ids.txt").write_text("a|some text\n\n")
    out = EV.run(str(tmp_path / "ref"), str(tmp_path / "syn"), EV.list_ids(str(tmp_path / "syn"), str(tmp_path / "ids.txt")),
                 n_cep=3, score=oracle_score(3))
    assert out["utterances"] == 1
    with pytest.raises(FileNotFoundError, match=r"missing file .*ref.mels.b\.npy"):
        EV.run(str(tmp_path / "ref"), str(tmp_path / "syn"), n_cep=3, score=oracle_score(3))


def test_command_without_pitch_or_energy_gives_null_figures(tmp_path):
    _tree(tmp_path / "ref", ["a"], [5], 0, pitch=False)
    _tree(tmp_path / "syn", ["a"], [5], 1)
    out = EV.run(str(tmp_path / "ref"), str(tmp_path / "syn"), n_cep=3, score=oracle_score(3))
    assert out["f0_rmse_cents"] is None and out["vuv_error"] is None and out["gpe"] is None and out["ffe"] is None
    assert out["energy_rmse"] is not None and out["mcd_db"] is not None
    _tree(tmp_path / "ref2", ["a"], [5], 0, energy=False)
    out = EV.run(str(tmp_path / "ref2"), str(tmp_path / "syn"), n_cep=3, score=oracle_score(3))
    assert out["energy_rmse"] is None and out["gpe"] is not None


def test_energy_length_must_match_the_mel(tmp_path):
    _tree(tmp_path / "ref", ["a"], [5], 0)
    _tree(tmp_path / "syn", ["a"], [5], 1)
    np.save(tmp_path / "syn" / "energy" / "a.npy", np.zeros(4, np.float32))
    with pytest.raises(ValueError, match="4 frames, its mel has 5"):
        EV.run(str(tmp_path / "ref"), str(tmp_path / "syn"), n_cep=3, score=oracle_score(3))


def test_command_batches_within_the_cell_budget(tmp_path):
    ids = [f"u{i}" for i in range(6)]
    _tree(tmp_path / "ref", ids, [10, 10, 20, 5, 5, 40], 0)
    _tree(tmp_path / "syn", ids, [10, 12, 20, 5, 6, 50], 1)
    log = []
    EV.run(str(tmp_path / "ref"), str(tmp_path / "syn"), n_cep=3, budget=450, score=oracle_score(3, log))
    # u0 + u1: 2 * 12 * 10 = 240; + u2 would be 3 * 20 * 20; u2 alone 400; + u3 = 800; u3 + u4 = 2 * 6 * 5; + u5 too big
    assert log == [["u0", "u1"], ["u2"], ["u3", "u4"], ["u5"]]


def test_command_line_parses_its_flags(tmp_path, capsys, monkeypatch):
    _tree(tmp_path / "ref", ["a"], [5], 0)
    _tree(tmp_path / "syn", ["a"], [6], 1)
    seen = {}

    def fake_backend(n_cep):
        seen["n_cep"] = n_cep
        return oracle_score(n_cep)
    monkeypatch.setattr(EV, "gpu_backend", fake_backend)
    EV.main(["--ref", str(tmp_path / "ref"), "--syn", str(tmp_path / "syn"), "--n-cep", "4", "--csv", str(tmp_path / "o.csv"),
             "--budget", "1000"])
    out = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert seen["n_cep"] == 4 and out["n_cep"] == 4 and out["utterances"] == 1
    assert os.path.exists(tmp_path / "o.csv")
