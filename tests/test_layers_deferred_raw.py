"""PoolLayer(DeferRelinearization=True) without a device: on the Raw backend (no ActivationConvDenseLayer) the layer applies its activation,
then itself, so the network computes exactly what the default one does; the configurations the deferred call cannot serve raise at
Prepare; and the C entry point is exported and bound."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _swap_squares(net, coeffs, W):
    from cryptonets_b200.layers import PolyActivation, SquareActivation
    layer = net
    while getattr(layer, "Source", None) is not None:
        if isinstance(layer.Source, SquareActivation):
            layer.Source = PolyActivation(Source=layer.Source.Source, Coefficients=coeffs, CoefficientScale=W)
        layer = layer.Source


@pytest.mark.parametrize("activation", ["square", "poly"])
def test_raw_backend_gives_the_default_scores(activation):
    from cryptonets_b200.networks import cryptonets_mnist, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    imgs = synthetic_mnist(16, seed=4)
    scores = []
    for defer in (False, True):
        net, _ = cryptonets_mnist(RawFactory(8192), imgs, timing=False, defer_relinearization=defer)
        if activation == "poly":
            _swap_squares(net, (0.25, 0.5, 0.125), 4.0)
        net.PrepareNetwork()
        out = net.GetNext()
        scores.append((np.asarray(out.Decrypt()), out.Scale))
    assert np.array_equal(scores[0][0], scores[1][0]) and scores[0][1] == scores[1][1]


def _dense(source, **kw):
    from cryptonets_b200.layers import PoolLayer
    return PoolLayer(Source=source, InputShape=[4], KernelShape=[4], Stride=[1000], MapCount=[2], Weights=np.arange(8.0), Bias=[1.0, 2.0],
                     DeferRelinearization=True, **kw)


def test_invalid_configurations_raise_at_prepare():
    from cryptonets_b200.layers import EncryptLayer, MatrixSource, PolyActivation, PoolLayer, SquareActivation
    from cryptonets_b200.raw import RawFactory
    enc = EncryptLayer(Source=MatrixSource(np.ones((2, 4))), Factory=RawFactory(8192))
    bad = {
        "unfused": _dense(SquareActivation(Source=enc), Fused=False),
        "not an activation": _dense(enc),
        "cubic": _dense(PolyActivation(Source=enc, Coefficients=(1.0, 0.0, 0.0, 1.0))),
        "quartic": _dense(PolyActivation(Source=enc, Coefficients=(1.0, 0.0, 0.0, 0.0, 1.0))),
        "mean pool": PoolLayer(Source=SquareActivation(Source=enc), InputShape=[4], KernelShape=[2], Stride=[2], DeferRelinearization=True),
    }
    for what, layer in bad.items():
        with pytest.raises(Exception, match="DeferRelinearization"):
            layer.PrepareNetwork()
    for ok in (_dense(SquareActivation(Source=enc)), _dense(PolyActivation(Source=enc, Coefficients=(1.0, 2.0, 3.0)))):
        ok.PrepareNetwork()
        assert ok.GetNext().RowCount == 2


def test_entry_point_is_exported_and_bound():
    from cryptonets_b200 import _lib
    assert "cnhe_layer_activation_conv_dense" in _lib.EXPORTS
    assert hasattr(_lib.lib(), "cnhe_layer_activation_conv_dense")
    with open(os.path.join(ROOT, "include", "cnhe.h")) as f:
        assert "int cnhe_layer_activation_conv_dense(" in f.read()
    with open(os.path.join(ROOT, "integration", "B200Native.cs")) as f:
        assert "cnhe_layer_activation_conv_dense(" in f.read()
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "check_csharp_bindings.py")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
