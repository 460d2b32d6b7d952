"""The diagonal (baby-step / giant-step) product's mathematics on the ciphertext's slot semantics, exact mod t, and the choice of the
number of baby steps.  CPU only: cryptonets_b200/diagonal.py restates what cnhe_diag_prepare / cnhe_mat_mul_diagonal compute."""
import numpy as np
import pytest

from cryptonets_b200 import diagonal as dg
from cryptonets_b200.interfaces import EVectorFormat
from cryptonets_b200.layers import LLDenseLayer, LLSingleLineReader
from cryptonets_b200.raw import RawFactory

T = 65537


def _matrix(rng, R, dim, t=T):
    return rng.integers(0, t, (R, dim)).astype(np.int64)


def _check(M, v, N, n1, t=T):
    d = dg.prerotated_diagonals(M, N, n1, t)
    y = dg.product(d, v, N, n1, t)
    R, dim = M.shape
    expect = np.zeros(N, np.int64)
    expect[:R] = (M.astype(object) @ np.asarray(v, dtype=object)) % t
    assert np.array_equal(y, expect)


def test_slot_rotations_act_on_two_rows():
    v = np.arange(8)
    assert list(dg.rotate_rows(v, 1)) == [1, 2, 3, 0, 5, 6, 7, 4]
    assert list(dg.rotate_columns(v)) == [4, 5, 6, 7, 0, 1, 2, 3]


@pytest.mark.parametrize("R", [1, 31, 35, 64])  # 1, N/2 - 1, N/2 + 3, N
@pytest.mark.parametrize("dim", [20, 32, 45, 64])  # inside the first row, exactly one row, into the second row, both rows
def test_product_equals_matrix_vector_n64(R, dim):
    N, rng = 64, np.random.default_rng(R * 100 + dim)
    M, v = _matrix(rng, R, dim), rng.integers(0, T, dim)
    for n1 in [1 << i for i in range(6)]:  # every power of two dividing N/2
        _check(M, v, N, n1)


@pytest.mark.parametrize("R", [1, 2047, 2051, 4096])
def test_product_equals_matrix_vector_n4096(R):
    N, rng = 4096, np.random.default_rng(R)
    dim = 2048 + 77  # crosses into the second row
    M = np.zeros((R, dim), np.int64)
    # a sparse matrix keeps the model fast; a dense band makes every diagonal class appear
    idx = rng.integers(0, R * dim, min(R * dim, 20000))
    M.flat[idx] = rng.integers(1, T, idx.size)
    v = rng.integers(0, T, dim)
    nz = dg.diagonal_flags(M, N)
    n1, _ = dg.plan_baby_steps(nz, N, dg.standard_galois_elts(N))
    for n1 in sorted({1, 2, 64, 2048, n1}):
        _check(M, v, N, n1)


def test_banded_matrix_drops_zero_diagonals():
    N, rng = 64, np.random.default_rng(3)
    M = np.zeros((32, 32), np.int64)
    for r in range(32):
        for off in (0, 3):
            M[r, (r + off) % 32] = rng.integers(1, T)
    nz = dg.diagonal_flags(M, N)
    assert sorted(zip(*np.nonzero(nz))) == [(0, 0), (0, 3)]
    d = dg.prerotated_diagonals(M, N, 4, T)
    assert sorted(d) == [(0, 0, 0), (0, 0, 3)]
    _check(M, rng.integers(0, T, 32), N, 4)


def test_hops_follow_the_galois_elements():
    N = 4096
    hops = dg.rotation_hops(N, dg.standard_galois_elts(N))
    assert [hops[s] for s in (1, 2, 3, 5, 7, 64, 1024, 2047)] == [1, 1, 2, 2, 2, 1, 1, 1]  # 2047 = 2048 - 1: the N/2 term is skipped
    assert dg.rotation_hops(N, dg.standard_galois_elts(N) + [pow(3, 7, 2 * N)])[7] == 1


@pytest.mark.parametrize("N,R,dim", [(4096, 2000, 4096), (4096, 1000, 1500), (16384, 5488, 16268), (16384, 2608, 11952)])
def test_planner_choice_is_the_cheapest(N, R, dim):
    # a dense R x dim matrix: every diagonal whose slots meet the matrix is nonzero
    half = N // 2
    nz = np.zeros((2, half), bool)
    nz[0, :] = True
    if dim > half:
        nz[1, :] = True
    n1, costs = dg.plan_baby_steps(nz, N, dg.standard_galois_elts(N))
    assert costs[n1] == min(costs.values())
    hops = dg.rotation_hops(N, dg.standard_galois_elts(N))
    nb = 2 if dim > half else 1
    assert costs[n1] == nb * sum(hops[1:n1]) + (nb - 1) + sum(hops[n1 * g] for g in range(1, half // n1))
    assert costs[n1] < 1000  # against 14 key switches per row on the row path


def _dense_layer(method, w, b, raw):
    src = LLSingleLineReader(raw, Scale=4.0, NormalizationFactor=1.0)
    layer = LLDenseLayer(Source=src, Weights=w.ravel(), Bias=b, WeightsScale=8.0, InputFormat=EVectorFormat.dense, ForceDenseFormat=True,
                         Method=method, Factory=RawFactory(64))
    layer.PrepareNetwork()
    return layer.GetNext().Decrypt(None)


def test_raw_backend_ignores_the_method():
    rng = np.random.default_rng(5)
    w, b, x = rng.normal(0, 1, (7, 40)), rng.normal(0, 1, 7), rng.normal(0, 1, (1, 40))
    assert np.array_equal(_dense_layer("rows", w, b, x), _dense_layer("diagonal", w, b, x))


def test_layer_refuses_bad_configurations():
    rng = np.random.default_rng(6)
    w, b, x = rng.normal(0, 1, (3, 8)), rng.normal(0, 1, 3), rng.normal(0, 1, (1, 8))
    for kw in (dict(Method="diagonal", ForceDenseFormat=False), dict(Method="diagonal", ForceDenseFormat=True, Shard=(0, 1, None)),
               dict(Method="columns", ForceDenseFormat=True)):
        layer = LLDenseLayer(Source=LLSingleLineReader(x, Scale=1.0, NormalizationFactor=1.0), Weights=w.ravel(), Bias=b, InputFormat=EVectorFormat.dense, Factory=RawFactory(64), **kw)
        with pytest.raises(Exception):
            layer.PrepareNetwork()
