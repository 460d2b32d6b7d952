"""cnhe_layer_square leaves its products unrelinearised until something reads them, and a scalar-MAC layer over such squares key-switches
its outputs instead of its inputs (DESIGN 4.15).  The words must be exactly those of the eager square followed by the same layer:

    sum_j W_mj relin(x_j) + bias = (sum_j W_mj (c0_j, c1_j) + bias) + sum_d S_md rlk_d,   S_md = sum_j W_mj digit_d(c2_j)

so every output here is compared word for word with the same layer over squares whose relinearisation was forced by a read (and, on
sampled outputs, with the CPU oracle's square + relinearise + scalar MAC).  The wgmma launcher reports on stderr which mode served a layer
("[umma digits" is the exact path)."""
import numpy as np
import pytest

from cryptonets_b200.engine import DENSE, SPARSE, Engine
from oracle.oracle_py import Oracle

pytestmark = pytest.mark.gpu

CTX = {
    4096: dict(t=[40961], dbc=10),
    8192: dict(t=[549764251649, 549764284417], dbc=10),
}
KERNEL_ENV = ("CNHE_MAC_NO_UMMA", "CNHE_MAC_NO_IMMA", "CNHE_MAC_INT", "CNHE_MUL_FUSED", "CNHE_KS_FUSED", "CNHE_NO_LAZY")


def _engine(N, monkeypatch, dbc=None, t=None):
    for var in KERNEL_ENV:
        monkeypatch.delenv(var, raising=False)
    cfg = CTX.get(N, dict(t=[786433], dbc=60))
    eng = Engine(t or cfg["t"], N, dbc or cfg["dbc"], 20, -1)
    eng.keygen(17)
    return eng


def _inputs(eng, n, dim, seed, bound=100):
    rng = np.random.default_rng(seed)
    return [eng.encrypt(rng.integers(-bound, bound, dim).astype(np.float64), 1.0, DENSE) for _ in range(n)]


def _layer(eng, rng, n_in, M, conv, wbound=120, big=False):
    if conv:  # convolution-shaped: a few taps per output, some padded
        K = 9
        g = rng.integers(-1, n_in, (M, K)).astype(np.int32)
        g[:, 0] = np.arange(M) % n_in
    else:
        K = n_in
        g = np.tile(np.arange(n_in, dtype=np.int32), (M, 1))
    w = rng.integers(-wbound, wbound + 1, (M, K))
    w[:, 0] = np.where(w[:, 0] == 0, 7, w[:, 0])
    if big:  # weights past a signed byte: the plan's W2 columns
        w[:, 1], w[:, 2] = 254, -254
    wv = [eng.plain(w[m].astype(np.float64), 1.0, SPARSE) for m in range(M)]
    bvals = [int(b) for b in rng.integers(-500, 500, M)]
    bias = [eng.plain(np.full(eng.N, float(b)), 1.0, DENSE) for b in bvals]
    return g, w, wv, bias, K, bvals


def _words(eng, vecs, blocks=1):
    return [np.stack([v.export_raw(ch, b) for ch in range(eng.P) for b in range(blocks)]) for v in vecs]


def _served(capfd):
    err = capfd.readouterr().err
    return "[umma digits" in err, "[umma " in err


def _run_both(eng, xs, g, wv, bias, M, K, monkeypatch, capfd):
    """the layer over pending squares, then over squares made eager by a read; returns (words, words, exact path served)"""
    monkeypatch.setenv("CNHE_UMMA_PROF", "1")
    capfd.readouterr()
    sq = eng.layer_square(xs)
    outs = eng.layer_conv_dense(sq, g, wv, bias, M, K)
    eng.sync()
    exact, _ = _served(capfd)
    sq2 = eng.layer_square(xs)
    sq2[-1].export_raw(0, 0)  # a read relinearises the whole group
    outs2 = eng.layer_conv_dense(sq2, g, wv, bias, M, K)
    eng.sync()
    exact2, _ = _served(capfd)
    assert not exact2
    # the squares the exact path read are still pending: read now, they give the eager words
    for a, b in zip(_words(eng, sq, xs[0].blocks), _words(eng, sq2, xs[0].blocks)):
        assert np.array_equal(a, b)
    return _words(eng, outs, xs[0].blocks), _words(eng, outs2, xs[0].blocks), exact, sq2


@pytest.mark.parametrize("N", [4096, 8192])
@pytest.mark.parametrize("shape", ["dense-10", "dense-100-w2", "conv-100"])
def test_exact_path_equals_eager_and_oracle(N, shape, monkeypatch, capfd):
    eng = _engine(N, monkeypatch)
    try:
        rng = np.random.default_rng(N + len(shape))
        M = 10 if shape == "dense-10" else 100
        n_in = 40
        xs = _inputs(eng, n_in, N, 3)
        g, w, wv, bias, K, bvals = _layer(eng, rng, n_in, M, shape.startswith("conv"), big=shape.endswith("w2"))
        got, want, exact, sq2 = _run_both(eng, xs, g, wv, bias, M, K, monkeypatch, capfd)
        assert exact, "the exact path did not serve the layer"
        for a, b in zip(got, want):
            assert np.array_equal(a, b)
        # the oracle: square, relinearise, scalar MAC, on sampled outputs of the first channel
        orc = Oracle(CTX[N]["t"][0], N, -1, CTX[N]["dbc"], 20)
        orc.keygen(17)
        t = CTX[N]["t"][0]
        sqw = []
        for i in range(n_in):
            x = xs[i].export_raw(0, 0)
            r = orc.relinearize(orc.multiply(x, x))
            if i < 3:
                assert np.array_equal(r, sq2[i].export_raw(0, 0))
            sqw.append(r)
        wres = np.array([[int(v) % t for v in row] for row in w], dtype=np.uint64)
        bres = np.array([b % t for b in bvals], dtype=np.uint64)
        ref = orc.mac_layer(np.stack(sqw), g, wres, bres, M, K, threads=8).reshape(M, -1)
        for m in (0, M // 2, M - 1):
            assert np.array_equal(ref[m], got[m][0]), m
    finally:
        eng.close()


def test_pending_read_by_every_kind_of_entry_point(monkeypatch):
    """a pending square read by decrypt, export, add, multiply_plain, rotate, square, poly2, copy, a row-major product or a one-output
    column-major product gives what the eager square gives; a pending square disposed unread frees its slab"""
    eng = _engine(4096, monkeypatch)
    try:
        N = eng.N
        xs = _inputs(eng, 4, N, 9, bound=30)
        ref = eng.layer_square(xs)
        ref[0].export_raw(0, 0)
        plain = eng.plain(np.arange(N, dtype=np.float64) % 7, 1.0, DENSE)
        one = eng.plain(np.array([3.0, -2.0, 5.0, 1.0]), 1.0, SPARSE)
        row = eng.plain(np.arange(N, dtype=np.float64) % 5, 1.0, DENSE)
        cases = {
            "decrypt": lambda v: eng.decrypt(v[0]),
            "export": lambda v: v[1].export_raw(0, 0),
            "add": lambda v: eng.add(v[0], v[1]).export_raw(0, 0),
            "multiply_plain": lambda v: eng.multiply_plain_many([v[2]], plain)[0].export_raw(0, 0),
            "rotate": lambda v: eng.rotate(v[3], 3).export_raw(0, 0),
            "square": lambda v: eng.layer_square([v[0]])[0].export_raw(0, 0),
            "poly2": lambda v: eng.layer_poly2([v[1]], eng.plain(np.array([2.0]), 1.0, SPARSE))[0].export_raw(0, 0),
            "copy": lambda v: eng.copy(v[2]).export_raw(0, 0),
            "colmajor": lambda v: eng.mat_mul_colmajor_sparse(v, one).export_raw(0, 0),
            "rowmajor": lambda v: eng.mat_mul_rowmajor([row], v[0], True).export_raw(0, 0),
        }
        for name, f in cases.items():
            want = f(ref)
            got = f(eng.layer_square(xs))
            assert np.array_equal(np.asarray(got), np.asarray(want)), name
        for _ in range(3):  # disposed unread: the group and its slab go with the last member
            eng.dispose_many(eng.layer_square(xs))
        assert np.array_equal(cases["export"](eng.layer_square(xs)), cases["export"](ref))
    finally:
        eng.close()


@pytest.mark.parametrize("decline", ["wide-weights", "trace_noise", "n16384", "two-blocks", "no-umma"])
def test_declines_give_eager_words(decline, monkeypatch, capfd):
    """layers the exact path cannot serve materialise their inputs and run as before, with the eager words"""
    N = 16384 if decline == "n16384" else 4096
    eng = _engine(N, monkeypatch)
    try:
        rng = np.random.default_rng(4)
        n_in, M = 24, 16
        dim = N + 9 if decline == "two-blocks" else N
        xs = _inputs(eng, n_in, dim, 6)
        g, w, wv, bias, K, _ = _layer(eng, rng, n_in, M, False, wbound=400 if decline == "wide-weights" else 120)
        if decline == "two-blocks":
            bias = None
        if decline == "trace_noise":
            eng.set_option("trace_noise", 1)
        if decline == "no-umma":
            monkeypatch.setenv("CNHE_MAC_NO_UMMA", "1")
        got, want, exact, _ = _run_both(eng, xs, g, wv, bias, M, K, monkeypatch, capfd)
        assert not exact
        for a, b in zip(got, want):
            assert np.array_equal(a, b)
    finally:
        eng.close()


def test_two_key_slots_then_per_client_layers(monkeypatch, capfd):
    """squares of two clients' vectors in one call, then one dense layer per client: each client's outputs equal its eager words"""
    eng = _engine(4096, monkeypatch)
    try:
        other = Engine([40961], 4096, 10, 20, -1)
        other.keygen(99)
        slot = eng.add_client_compact(other.save_compact_keys())
        rng = np.random.default_rng(8)
        n_in, M = 20, 12
        xs = _inputs(eng, n_in, eng.N, 1) + _inputs(eng, n_in, eng.N, 2)
        for v in xs[n_in:]:
            v.set_key_slot(slot)
        g, w, wv, bias, K, _ = _layer(eng, rng, n_in, M, False)
        monkeypatch.setenv("CNHE_UMMA_PROF", "1")
        capfd.readouterr()
        sq = eng.layer_square(xs)
        outs = [eng.layer_conv_dense(sq[:n_in], g, wv, bias, M, K), eng.layer_conv_dense(sq[n_in:], g, wv, bias, M, K)]
        eng.sync()
        assert _served(capfd)[0]
        sq2 = eng.layer_square(xs)
        sq2[0].export_raw(0, 0)
        outs2 = [eng.layer_conv_dense(sq2[:n_in], g, wv, bias, M, K), eng.layer_conv_dense(sq2[n_in:], g, wv, bias, M, K)]
        for o, o2 in zip(outs, outs2):
            for a, b in zip(_words(eng, o), _words(eng, o2)):
                assert np.array_equal(a, b)
        other.close()
    finally:
        eng.close()
