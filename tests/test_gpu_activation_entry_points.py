"""Rules of the activation entry points that their word-for-word tests do not reach: cnhe_layer_square takes inputs of different scales,
and a square of pending squares is relinearised at once rather than left pending (DESIGN 4.15)."""
import numpy as np
import pytest

from cryptonets_b200.engine import DENSE, SPARSE, Engine

pytestmark = pytest.mark.gpu

KERNEL_ENV = ("CNHE_MAC_NO_UMMA", "CNHE_MAC_NO_IMMA", "CNHE_MAC_INT", "CNHE_MUL_FUSED", "CNHE_KS_FUSED")


def _engine(monkeypatch):
    for var in KERNEL_ENV:
        monkeypatch.delenv(var, raising=False)
    eng = Engine([40961], 4096, 10, 20, -1)
    eng.keygen(17)
    return eng


def test_square_takes_inputs_of_two_scales(monkeypatch):
    """each output at its own input's scale squared: the pending square, then the eager square of squares"""
    eng = _engine(monkeypatch)
    try:
        rng = np.random.default_rng(1)
        vals = [rng.integers(-3, 4, eng.N).astype(np.float64) for _ in range(2)]
        xs = [eng.encrypt(vals[0], 1.0, DENSE), eng.encrypt(vals[1], 2.0, DENSE)]
        sq = eng.layer_square(xs)
        assert [o.scale for o in sq] == [1.0, 4.0]
        q4 = eng.layer_square(sq)
        assert [o.scale for o in q4] == [1.0, 16.0]
        for v, s, f in zip(vals, sq, q4):
            assert np.array_equal(eng.decrypt(s), v ** 2) and np.array_equal(eng.decrypt(f), v ** 4)
    finally:
        eng.close()


def test_square_of_pending_squares_is_relinearised(monkeypatch, capfd):
    """a dense layer over pending squares takes the exact path ("[umma digits" on stderr); over squares of those squares, a polynomial
    chain that the square relinearises at once, it takes the ordinary one"""
    eng = _engine(monkeypatch)
    try:
        rng = np.random.default_rng(2)
        n_in, M = 40, 10
        xs = [eng.encrypt(rng.integers(-3, 4, eng.N).astype(np.float64), 1.0, DENSE) for _ in range(n_in)]
        g = np.tile(np.arange(n_in, dtype=np.int32), (M, 1))
        wv = [eng.plain(rng.integers(1, 120, n_in).astype(np.float64), 1.0, SPARSE) for _ in range(M)]
        monkeypatch.setenv("CNHE_UMMA_PROF", "1")
        exact = []
        for make in (lambda: eng.layer_square(xs), lambda: eng.layer_square(eng.layer_square(xs))):
            capfd.readouterr()
            eng.layer_conv_dense(make(), g, wv, None, M, n_in)
            eng.sync()
            exact.append("[umma digits" in capfd.readouterr().err)
        assert exact == [True, False], exact
    finally:
        eng.close()
