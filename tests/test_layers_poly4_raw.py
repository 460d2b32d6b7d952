"""PolyActivation with 4 or 5 coefficients (the cubic and quartic of cnhe_layer_poly) on the Raw backend: the rounded integer polynomial,
evaluated exactly, its output scale W s^d, the coefficient-scale checks and refusals, and ApplyBatch."""
import numpy as np
import pytest

from cryptonets_b200.interfaces import EVectorFormat
from cryptonets_b200.layers import MatrixSource, PolyActivation
from cryptonets_b200.raw import RawFactory, RawMatrix, poly_scale


def _layer(x, s, coeffs, W):
    src = MatrixSource(x, Scale=s)
    layer = PolyActivation(Source=src, Coefficients=coeffs, CoefficientScale=W)
    layer.Prepare()
    return src, layer


def _want(xi, coeffs, W, s):
    d = len(coeffs) - 1
    ints = [int(np.rint(c * poly_scale(W, s, i))) for i, c in enumerate(coeffs)]  # highest degree first
    acc = np.zeros(xi.shape, dtype=object)
    for v in ints:
        acc = acc * xi.astype(np.int64).astype(object) + v
    return np.array(acc.tolist(), dtype=np.float64), poly_scale(W, s, d)


CASES = [((0.0625, 0.0, 0.5, 0.25, 0.125), 16.0),       # a quartic ReLU-style fit, no cubic term
         ((-0.02, 0.13, -0.7, 1.9, -3.1), 100.0),        # negative coefficients
         ((1.0, 0.0, 0.0, 0.0, 0.0), 1.0),               # x^4
         ((0.004, 0.0, 0.5, 0.5), 256.0),                # an odd cubic (sigmoid-style)
         ((-1.5, 0.25, -0.125, 7.0), 8.0)]


@pytest.mark.parametrize("coeffs, W", CASES)
def test_poly_activation_degree_3_and_4_matches_integer_polynomial(coeffs, W):
    rng = np.random.default_rng(5)
    s = 8.0
    x = rng.integers(-60, 60, (7, 4)) / s
    src, layer = _layer(x, s, coeffs, W)
    out = layer.Apply(src.GetNext())
    want, scale = _want(np.rint(x * s), coeffs, W, s)
    assert layer.GetOutputScale() == scale == W * s ** (len(coeffs) - 1)
    assert out.Scale == scale
    assert np.array_equal(out.Data, want)


def test_terms_past_2_53_are_exact_before_the_final_rounding():
    s, W = 1024.0, 1024.0
    x = np.array([[1000.0, -999.0]])  # x s ~ 2^20: x^4 s^4 W ~ 2^90
    src, layer = _layer(x, s, (1.0, 0.0, 0.0, 0.0, 3.0), W)
    out = layer.Apply(src.GetNext())
    xi = [int(v) for v in np.rint(x * s).reshape(-1)]
    c0 = int(np.rint(3.0 * W * s ** 4))
    assert out.Data.reshape(-1).tolist() == [float(int(W) * v ** 4 + c0) for v in xi]


def test_coefficients_that_round_to_zero_are_left_out_but_the_leading_one_stays():
    s, W = 4.0, 2.0
    src, layer = _layer(np.array([[1.0]]), s, (0.5, 0.0, 0.1, 0.001, 1.0), W)  # 0.001 W s^3 rounds to 0
    vs = layer.coefficientVectors
    assert len(vs) == 5 and vs[0] is not None and vs[1] is None and vs[3] is None
    assert vs[2] is not None and vs[4] is not None


def test_scales_refused_like_the_c_abi():
    f = RawFactory(8192)
    m = RawMatrix(np.array([[1.0, 2.0]]), 2.0, None, 8192)  # s = 2
    W = 3.0
    ok = [f.GetPlainVector([1.0], EVectorFormat.sparse, poly_scale(W, 2.0, i)) for i in range(5)]
    assert m.PolyActivation(ok).Scale == poly_scale(W, 2.0, 4)
    assert m.PolyActivation(ok[:4]).Scale == poly_scale(W, 2.0, 3)
    bad = list(ok)
    bad[2] = f.GetPlainVector([1.0], EVectorFormat.sparse, poly_scale(W, 2.0, 3))  # x^2 term at W s^3 instead of W s^2
    with pytest.raises(Exception, match="Scales do not match"):
        m.PolyActivation(bad)
    with pytest.raises(Exception, match="leading coefficient"):
        m.PolyActivation([None] + ok[1:])
    with pytest.raises(Exception, match="degree"):
        m.PolyActivation(ok + ok[:1])
    with pytest.raises(Exception):
        m.PolyActivation(ok, ok[0])  # a list takes no b or c


def test_wrong_length_is_refused():
    src = MatrixSource(np.array([[1.0]]), Scale=1.0)
    layer = PolyActivation(Source=src, Coefficients=(1.0, 2.0), CoefficientScale=1.0)
    with pytest.raises(Exception, match="3, 4 or 5"):
        layer.Prepare()


def test_length_3_keeps_the_quadratic():
    s, W = 16.0, 8.0
    src, layer = _layer(np.array([[0.5, -1.0]]), s, (0.125, 0.5, 0.25), W)
    assert len(layer.coefficientVectors) == 3 and layer.GetOutputScale() == W * s * s
    out = layer.Apply(src.GetNext())
    xi = np.array([8.0, -16.0])
    assert np.array_equal(out.Data.reshape(-1), 1 * xi * xi + 64 * xi + 512)


def test_apply_batch_equals_apply():
    s, W = 4.0, 2.0
    rng = np.random.default_rng(9)
    xs = [rng.integers(-20, 20, (3, 2)) / s for _ in range(3)]
    src, layer = _layer(xs[0], s, (0.25, -0.5, 0.0, 1.0, 2.0), W)
    ms = [RawMatrix(x, s, None, 8192) for x in xs]
    batch = layer.ApplyBatch(ms)
    for m, b in zip(ms, batch):
        assert np.array_equal(layer.Apply(m).Data, b.Data)
