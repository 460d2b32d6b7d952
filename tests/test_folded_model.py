"""The folded diagonal product (cnhe_diag_prepare_folded, DESIGN.md section 4.10) without a GPU: the exact mod-t model of
cryptonets_b200/diagonal.py against M v, its planner against a brute-force count of the rotations, and LLDenseLayer.Method = "folded" on
the Raw backend."""
import numpy as np
import pytest

from cryptonets_b200 import diagonal as dg
from cryptonets_b200 import networks as nw
from cryptonets_b200.interfaces import EVectorFormat
from cryptonets_b200.layers import LLDenseLayer, LLSingleLineReader
from cryptonets_b200.raw import RawFactory

T = 65537


def _pow2_upto(n):
    return [1 << i for i in range(n.bit_length()) if 1 << i <= n]


def _cases(N):
    half = N // 2
    for dim in (half // 2 + 3, half, half + 7, N):
        for W in _pow2_upto(half):
            for R in sorted({1, 3, W - 1, W}):
                if 1 <= R <= W:
                    yield dim, W, R


@pytest.mark.parametrize("N", [64, 4096])
def test_folded_model_equals_matrix_product(N):
    rng = np.random.default_rng(N)
    for dim, W, R in _cases(N):
        M = rng.integers(0, T, (R, dim))
        v = rng.integers(0, T, dim)
        want = [int(x) for x in (M.astype(object) @ v.astype(object)) % T]
        # every n1 at the small ring; at N = 4096 the extremes and one in between (each n1 is a different split of the same sum)
        n1s = _pow2_upto(W) if N == 64 else sorted({1, _pow2_upto(max(1, int(W ** 0.5)))[-1], W})
        for n1 in n1s:
            y = dg.folded_product(dg.folded_diagonals(M, N, W, n1, T), v, N, W, n1, R, dim, T)
            assert [int(x) for x in y[:R]] == want, (N, dim, W, R, n1)
            assert not y[R:].any(), (N, dim, W, R, n1)


def _nonzero_wrapped(M, N, W):
    """The j < W whose wrapped diagonal E_j[(a, x)] = M[x mod W, a N/2 + (x + j mod N/2)] has a nonzero weight, from the definition."""
    half = N // 2
    R, dim = M.shape
    Mt = np.zeros((W, N), dtype=np.int64)
    Mt[:R, :dim] = M
    i = np.arange(N)
    a, x = i // half, i % half
    return [j for j in range(W) if Mt[x % W, a * half + (x + j) % half].any()]


def _brute_force_plan(M, N, elts):
    """(W, n1, key switches) counted from the nonzero wrapped diagonals: rotate_rows(h) for every baby step h != 0 and rotate_rows(n1 g)
    for every giant step g != 0 one of them uses (their hops), the column fold when dim > N/2, one hop per row fold."""
    half = N // 2
    R, dim = M.shape
    hops = dg.rotation_hops(N, elts)
    best = None
    for W in [w for w in _pow2_upto(half) if w >= R]:
        js = _nonzero_wrapped(M, N, W)
        folds = half.bit_length() - W.bit_length()
        for n1 in _pow2_upto(W):
            cost = sum(hops[h] for h in {j % n1 for j in js} if h) + sum(hops[n1 * g] for g in {j // n1 for j in js} if g)
            cost += (1 if dim > half else 0) + folds
            if best is None or (cost, W, n1) < (best[2], best[0], best[1]):
                best = (W, n1, cost)
    return best


def test_planner_lola_small_score_layer():
    M = np.asarray(nw.lola_small_weights()["Weights_1"]).reshape(10, -1)
    assert M.shape == (10, 845)
    N = 8192
    elts = dg.standard_galois_elts(N)
    assert dg.plan_folded(M, N, elts) == (16, 4, 16)
    assert _brute_force_plan(M, N, elts) == (16, 4, 16)  # against 10 x 13 = 130 on the rows method


@pytest.mark.parametrize("N,R,dim,density", [(64, 3, 40, 1.0), (64, 5, 20, 0.2), (256, 10, 200, 1.0), (256, 2, 30, 0.05),
                                             (1024, 10, 845, 1.0), (1024, 7, 1000, 0.02)])
def test_planner_matches_brute_force(N, R, dim, density):
    rng = np.random.default_rng(R * dim)
    M = rng.integers(1, T, (R, dim)) * (rng.random((R, dim)) < density)
    elts = dg.standard_galois_elts(N)
    assert dg.plan_folded(M, N, elts) == _brute_force_plan(M, N, elts)


@pytest.mark.parametrize("shape,N", [((10, 5488), 16384), ((10, 2608), 16384)])
def test_planner_score_layers_of_cifar_and_large(shape, N):
    rng = np.random.default_rng(1)
    M = rng.integers(1, T, shape)
    W, n1, cost = dg.plan_folded(M, N, dg.standard_galois_elts(N))
    assert W >= 10 and W % n1 == 0
    assert cost <= 18  # against 10 x 14 = 140 on the rows method


def _layer(w, b, x, **kw):
    layer = LLDenseLayer(Source=LLSingleLineReader(x, Scale=4.0, NormalizationFactor=1.0), Weights=w.ravel(), Bias=b, WeightsScale=8.0,
                         Factory=RawFactory(64), **kw)
    layer.PrepareNetwork()
    return layer


@pytest.mark.parametrize("force", [False, True])
def test_raw_folded_layer_is_dense_matrix_product(force):
    rng = np.random.default_rng(11)
    w, b, x = rng.integers(-9, 9, (7, 40)).astype(float), rng.integers(-9, 9, 7).astype(float), rng.integers(-9, 9, (1, 40)).astype(float)
    layer = _layer(w, b, x, InputFormat=EVectorFormat.dense, ForceDenseFormat=force, Method="folded")
    out = layer.GetNext()
    col = out.GetColumn(0)
    assert col.Format == EVectorFormat.dense and col.Dim == 7
    assert np.array_equal(np.asarray(out.Decrypt(None)).reshape(-1), w @ x[0] + b)


def test_raw_lola_small_folded_scores_equal_rows():
    imgs = nw.synthetic_mnist(2, seed=4)
    got = []
    for method in ("rows", "folded"):
        net, _ = nw.lola_small(RawFactory(8192), imgs, dense_method=method)
        net.PrepareNetwork()
        got.append(np.asarray(net.GetNext().Decrypt(None)))
    assert np.array_equal(got[0], got[1])


@pytest.mark.parametrize("kw", [dict(InputFormat=EVectorFormat.sparse, Method="folded"),
                                dict(InputFormat=EVectorFormat.dense, Method="folded", Shard=(0, 1, None)),
                                dict(InputFormat=EVectorFormat.dense, Method="diagonal", ForceDenseFormat=False)])
def test_layer_refuses_bad_configurations(kw):
    rng = np.random.default_rng(6)
    w, b, x = rng.normal(0, 1, (3, 8)), rng.normal(0, 1, 3), rng.normal(0, 1, (1, 8))
    with pytest.raises(Exception):
        _layer(w, b, x, **kw)


def test_folded_accepts_ntt_bytes():
    rng = np.random.default_rng(7)
    w, b, x = rng.integers(-9, 9, (3, 8)).astype(float), rng.integers(-9, 9, 3).astype(float), rng.integers(-9, 9, (1, 8)).astype(float)
    layer = _layer(w, b, x, InputFormat=EVectorFormat.dense, Method="folded", DiagonalNttBytes=None)
    assert np.array_equal(np.asarray(layer.GetNext().Decrypt(None)).reshape(-1), w @ x[0] + b)
