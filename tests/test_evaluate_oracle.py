"""The float64 evaluation oracle (oracle/eval_oracle.py) on its own: the anti-diagonal DTW against a plain double loop,
the DCT basis against scipy, exact zeros on identical inputs, a hand-worked case that pins the tie order, and the prosody
sums on a crafted path."""
import math

import numpy as np
import pytest
import scipy.fft

from fastspeech2_b200.evaluate import MCD_SCALE, dct_basis
from oracle import eval_oracle as E


def brute_dtw(cx, cy):
    """Row-major double loop in pure Python floats: the definition, one cell at a time."""
    Lx, Ly, K = len(cx), len(cy), len(cx[0])
    A = [[0.0] * Ly for _ in range(Lx)]
    back = [[None] * Ly for _ in range(Lx)]
    for i in range(Lx):
        for j in range(Ly):
            acc = 0.0
            for k in range(K):
                diff = float(cx[i][k]) - float(cy[j][k])
                acc = acc + diff * diff
            d = math.sqrt(acc)
            best, arg = None, None
            for pi, pj in ((i - 1, j - 1), (i - 1, j), (i, j - 1)):
                if pi >= 0 and pj >= 0 and (best is None or A[pi][pj] < best):
                    best, arg = A[pi][pj], (pi, pj)
            A[i][j] = d if best is None else d + best
            back[i][j] = arg
    path, c = [], (Lx - 1, Ly - 1)
    while c is not None:
        path.append(c)
        c = back[c[0]][c[1]]
    return A[Lx - 1][Ly - 1], path[::-1]


@pytest.mark.parametrize("seed", range(6))
def test_diagonal_dtw_matches_the_double_loop(seed):
    rng = np.random.default_rng(seed)
    Lx, Ly, K = rng.integers(1, 23), rng.integers(1, 23), int(rng.integers(1, 6))
    cx, cy = rng.standard_normal((Lx, K)), rng.standard_normal((Ly, K))
    if seed % 2:      # coarse values make ties common
        cx, cy = np.round(cx * 2) / 2, np.round(cy * 2) / 2
    cost, path, _ = E.dtw(cx, cy)
    want_cost, want_path = brute_dtw(cx.tolist(), cy.tolist())
    assert np.float64(cost).tobytes() == np.float64(want_cost).tobytes()
    assert [tuple(p) for p in path.tolist()] == want_path


def test_dct_basis_is_scipys_orthonormal_dct_ii_without_c0():
    for M, K in ((80, 24), (80, 79), (16, 1), (7, 6)):
        want = scipy.fft.dct(np.eye(M), type=2, norm="ortho", axis=1)[:, 1:K + 1]
        np.testing.assert_allclose(dct_basis(M, K), want, rtol=0, atol=1e-14)
    assert MCD_SCALE == E.MCD_SCALE == 10.0 * math.sqrt(2.0) / math.log(10.0)


def test_identical_sequences_give_zero_on_the_diagonal():
    rng = np.random.default_rng(3)
    mel = rng.uniform(-11, 2, (37, 80)).astype(np.float32)
    r = E.evaluate_pair(mel, mel, dct_basis(80, 24))
    assert r["mcd"] == 0.0 and r["cost"] == 0.0 and r["plen"] == 37
    assert r["path"].tolist() == [[t, t] for t in range(37)]


def test_hand_worked_three_by_four_pins_the_tie_order():
    # d = |cx - cy|:  [[0, 1, 1, 2], [2, 1, 1, 0], [2, 1, 1, 0]]
    # A = [[0, 1, 2, 4], [2, 1, 2, 2], [4, 2, 2, 2]]; A(1,2), A(1,3) and A(2,3) tie their diagonal with others and take it
    cx, cy = np.array([[0.0], [2.0], [2.0]]), np.array([[0.0], [1.0], [1.0], [2.0]])
    cost, path, A = E.dtw(cx, cy)
    np.testing.assert_array_equal(A, [[0, 1, 2, 4], [2, 1, 2, 2], [4, 2, 2, 2]])
    assert cost == 2.0
    assert path.tolist() == [[0, 0], [0, 1], [1, 2], [2, 3]]
    assert E.mcd(cost, len(path)) == (2.0 / 4.0) * MCD_SCALE


def test_prosody_on_a_crafted_path():
    path = np.array([[0, 0], [1, 0], [2, 1], [2, 2], [3, 3]])
    f0x = np.array([100.0, 0.0, 130.0])             # plens_x = 3 < Lx = 4: frame 3 counts as unvoiced
    f0y = np.array([100.0, 110.0, 100.0, 100.0])
    ex, ey = np.array([1, 2, 3, 4], np.float32), np.ones(4, np.float32)
    counts, sums = E.prosody(path, f0x, f0y, ex, ey)
    assert counts == (5, 2, 3, 1)                    # (1,0) and (3,3) differ; (2,2) has |1.3 - 1| > 0.2, (2,1) does not
    c1 = 1200.0 * np.log2(np.float64(130.0) / np.float64(110.0))
    c2 = 1200.0 * np.log2(np.float64(130.0) / np.float64(100.0))
    assert sums[0] == (0.0 + c1 * c1) + c2 * c2
    assert sums[1] == 18.0
