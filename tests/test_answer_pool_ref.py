"""The numpy reference of the answer-pool top-k (tests/pool_topk_ref.py), pinned on hand cases: ties across the device
routes' chunk and tile boundaries (64-column tiles, 256-row chunks), k = m, duplicate scores."""
import numpy as np
import pytest

from pool_topk_ref import pool_topk, topk_rows


def test_hand_cases():
    s = np.array([[1, 3, 3, 2, 3],
                  [0, 0, 0, 0, 0],
                  [5, 4, 3, 2, 1]], np.float64)
    i, v = topk_rows(s, 3)
    assert i.tolist() == [[1, 2, 4], [0, 1, 2], [0, 1, 2]]
    assert v.tolist() == [[3, 3, 3], [0, 0, 0], [5, 4, 3]]


def test_k_equals_m_is_a_stable_sort():
    s = np.array([[2, -1, 2, 7, -1, 0]], np.float64)
    i, v = topk_rows(s, 6)
    assert i.tolist() == [[3, 0, 2, 5, 1, 4]]
    assert v.tolist() == [[7, 2, 2, 0, -1, -1]]


@pytest.mark.parametrize("edge", [63, 64, 255, 256])
def test_ties_across_boundaries(edge):
    m = 600
    s = np.zeros((2, m))
    s[0, [edge, edge + 1, edge - 1, 5, m - 1]] = 9.0        # five equal maxima on both sides of a tile / chunk edge
    s[1, :] = 1.0
    s[1, [m - 1, 0]] = 2.0
    i, v = topk_rows(s, 4)
    assert i[0].tolist() == sorted([edge, edge + 1, edge - 1, 5, m - 1])[:4]
    assert (v[0] == 9.0).all()
    assert i[1].tolist() == [0, m - 1, 1, 2]


def test_duplicate_rows_come_back_adjacent():
    rng = np.random.default_rng(0)
    E = rng.integers(-2, 3, (40, 8)).astype(np.float64)
    E = np.concatenate([E, E[[3, 17]]])                    # rows 40, 41 duplicate rows 3, 17
    Q = rng.integers(-2, 3, (50, 8)).astype(np.float64)
    i, v = pool_topk(Q, E, 42, chunk=7)
    for r in range(len(Q)):
        for a, b in ((3, 40), (17, 41)):
            pa, pb = list(i[r]).index(a), list(i[r]).index(b)
            assert v[r, pa] == v[r, pb] and pb > pa
        assert all((v[r, j] > v[r, j + 1]) or (v[r, j] == v[r, j + 1] and i[r, j] < i[r, j + 1]) for j in range(41))


def test_chunked_equals_whole():
    rng = np.random.default_rng(1)
    Q = rng.integers(-2, 3, (300, 16))
    E = rng.integers(-2, 3, (1000, 16))
    a = pool_topk(Q, E, 32, chunk=300)
    b = pool_topk(Q, E, 32, chunk=13)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
