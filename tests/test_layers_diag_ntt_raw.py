"""LLDenseLayer.DiagonalNttBytes on the Raw backend: validated with the other method checks, and ignored by the computation."""
import numpy as np
import pytest

from cryptonets_b200 import networks as nw
from cryptonets_b200.raw import RawFactory


def _scores(build, imgs, **kw):
    net, _ = build(RawFactory(16384), imgs, **kw)
    net.PrepareNetwork()
    return np.asarray(net.GetNext().Decrypt()).reshape(-1)


@pytest.mark.parametrize("budget", [1, 3 << 30, None])
def test_ntt_bytes_needs_the_diagonal_method(budget):
    with pytest.raises(Exception, match="DiagonalNttBytes"):
        _scores(nw.lola_large, nw.synthetic_mnist(1, seed=3), dense_method="rows", diag_ntt_bytes=budget)


@pytest.mark.parametrize("budget", [-1, 1 << 64])
def test_ntt_bytes_out_of_range(budget):
    with pytest.raises(Exception, match="DiagonalNttBytes"):
        _scores(nw.lola_large, nw.synthetic_mnist(1, seed=3), dense_method="diagonal", diag_ntt_bytes=budget)


def test_raw_output_ignores_the_budget():
    imgs = nw.synthetic_mnist(1, seed=3)
    want = _scores(nw.lola_large, imgs, dense_method="diagonal")
    for budget in (3 << 30, None):
        assert np.array_equal(_scores(nw.lola_large, imgs, dense_method="diagonal", diag_ntt_bytes=budget), want)
    assert np.array_equal(_scores(nw.lola_large, imgs), want)
