"""PolyActivation (a x^2 + b x + c) on the Raw backend against numpy: integer coefficients, output scale, rounding of negative
coefficients, coefficients that round to zero, and ApplyBatch."""
import numpy as np
import pytest

from cryptonets_b200.interfaces import EMatrixFormat, EVectorFormat
from cryptonets_b200.layers import EncryptLayer, MatrixSource, PolyActivation, SquareActivation
from cryptonets_b200.networks import lola_small, serve_batch, synthetic_mnist
from cryptonets_b200.raw import RawFactory, RawMatrix


def _layer(x, s, coeffs, W):
    src = MatrixSource(x, Scale=s)
    layer = PolyActivation(Source=src, Coefficients=coeffs, CoefficientScale=W)
    layer.Prepare()
    return src, layer


@pytest.mark.parametrize("coeffs, W", [((0.125, 0.5, 0.25), 8.0), ((-0.3, -1.7, -2.45), 10.0), ((0.0937, -0.51, 0.3), 64.0), ((1.0, 0.0, 0.0), 1.0)])
def test_poly_activation_matches_numpy(coeffs, W):
    rng = np.random.default_rng(3)
    s = 16.0
    x = rng.integers(-40, 40, (6, 5)) / s
    src, layer = _layer(x, s, coeffs, W)
    out = layer.Apply(src.GetNext())
    xi = np.rint(x * s)
    a, b, c = coeffs
    A, B, C = np.rint(a * W), np.rint(b * W * s), np.rint(c * W * s * s)  # Math.Round, ties to even; negatives round symmetrically
    want = A * xi * xi + B * xi + C
    assert layer.GetOutputScale() == W * s * s
    assert out.Scale == W * s * s
    assert np.array_equal(out.Data, want)
    assert np.array_equal(out.Decrypt(), want / (W * s * s))


def test_negative_coefficients_round_like_plain_vectors():
    s, W = 4.0, 2.0
    src, layer = _layer(np.array([[1.0, -2.0]]), s, (-1.25, -0.3125, -0.03125), W)  # -2.5, -2.5, -1.0 before rounding
    A, B, C = (v.Data[0] for v in layer.coefficientVectors)
    assert (A, B, C) == (-2.0, -2.0, -1.0)  # ties to even, as the encoders round
    out = layer.Apply(src.GetNext())
    xi = np.array([[4.0, -8.0]])
    assert np.array_equal(out.Data, -2 * xi * xi - 2 * xi - 1)


def test_zero_terms_are_left_out():
    src, layer = _layer(np.ones((2, 2)), 8.0, (0.5, 0.01, 0.001), 4.0)  # A = 2, B = round(0.32) = 0, C = round(0.256) = 0
    assert layer.coefficientVectors[1] is None and layer.coefficientVectors[2] is None
    out = layer.Apply(src.GetNext())
    assert np.array_equal(out.Data, np.full((2, 2), 2 * 64.0))
    assert out.Scale == 4.0 * 64


def test_apply_batch_equals_apply_per_matrix():
    rng = np.random.default_rng(5)
    s = 16.0
    src, layer = _layer(np.zeros((1, 1)), s, (0.2, -0.7, 1.3), 32.0)
    ms = [RawMatrix(rng.integers(-30, 30, (7, 3)) / s, s, EMatrixFormat.ColumnMajor, 8192) for _ in range(3)]
    batched = layer.ApplyBatch(ms)
    assert len(batched) == 3
    for m, o in zip(ms, batched):
        assert np.array_equal(o.Data, layer.Apply(m).Data)
        assert o.Scale == layer.GetOutputScale()


def test_lola_small_with_poly_activation_serves_a_batch():
    """lola_small with its square replaced: serve_batch takes the layer like SquareActivation, and (1, 0, 0) at W = 1 is the square."""
    imgs = synthetic_mnist(2, seed=9)
    outs = {}
    for coeffs in ((1.0, 0.0, 0.0), (0.25, 0.5, 0.125)):
        f = RawFactory(8192)
        net, reader = lola_small(f, imgs)
        sq = net.Source
        assert isinstance(sq, SquareActivation)
        net.Source = PolyActivation(Source=sq.Source, Coefficients=coeffs, CoefficientScale=4.0 if coeffs[1] else 1.0)
        layer = net
        while not isinstance(layer, EncryptLayer):
            layer = layer.Source
        ms = [layer.Apply(reader.GetNext()) for _ in range(len(imgs))]
        outs[coeffs] = [np.asarray(o.Decrypt()) for o in serve_batch(net, ms)]
        assert net.Source.GetOutputScale() == net.Source.CoefficientScale * net.Source.Source.GetOutputScale() ** 2
    f = RawFactory(8192)
    net, reader = lola_small(f, imgs)
    enc = net.Source
    while not isinstance(enc, EncryptLayer):
        enc = enc.Source
    want = [np.asarray(o.Decrypt()) for o in serve_batch(net, [enc.Apply(reader.GetNext()) for _ in range(len(imgs))])]
    for a, b in zip(outs[(1.0, 0.0, 0.0)], want):
        assert np.array_equal(a, b)
    assert not all(np.array_equal(a, b) for a, b in zip(outs[(0.25, 0.5, 0.125)], want))


def test_raw_twin_refuses_mismatched_coefficient_scales():
    """the Raw twin checks the coefficient scales exactly as cnhe_layer_poly2 does: scale(b) s and scale(c) must equal scale(a) s^2"""
    f = RawFactory(8192)
    s = 4.0
    m = RawMatrix(np.ones((3, 2)), s, EMatrixFormat.ColumnMajor, 8192)
    a = f.GetPlainVector([1.0], EVectorFormat.sparse, 2.0)
    good_b, good_c = f.GetPlainVector([1.0], EVectorFormat.sparse, 8.0), f.GetPlainVector([1.0], EVectorFormat.sparse, 32.0)
    assert m.PolyActivation(a, good_b, good_c).Scale == 32.0
    for b, c in ((f.GetPlainVector([1.0], EVectorFormat.sparse, 2.0), None), (None, f.GetPlainVector([1.0], EVectorFormat.sparse, 8.0))):
        with pytest.raises(Exception, match="Scales do not match"):
            m.PolyActivation(a, b, c)
