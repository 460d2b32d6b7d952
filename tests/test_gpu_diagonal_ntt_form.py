"""Diagonal matrices held in NTT form (cnhe_diag_prepare_ntt): the resident words against the oracle's lift and forward transform, the
product word for word against the coefficient-form matrix of the same rows for every budget, client count, key-slot mix and the integer
path, the budget bookkeeping, the refusals (the removed MAC option among them), and LoLa-Large / LoLa-CIFAR with a partial
budget."""
import os

import numpy as np
import pytest

from cryptonets_b200 import diagonal as dg
from cryptonets_b200._lib import CnheError

pytestmark = pytest.mark.gpu

ERR_INVALID = -1
T, N = 40961, 4096
ALL = None  # Engine.diag_prepare's ntt_bytes for the whole matrix


def _engine(t=T, n=N, int_path=False, seed=1234):
    from cryptonets_b200.engine import Engine
    saved = os.environ.pop("CNHE_NTT_INT", None)
    if int_path:
        os.environ["CNHE_NTT_INT"] = "1"
    try:
        eng = Engine([t], n, 10, 20, -1)
    finally:
        os.environ.pop("CNHE_NTT_INT", None)
        if saved is not None:
            os.environ["CNHE_NTT_INT"] = saved
    eng.keygen(seed)
    return eng


@pytest.fixture(scope="module")
def eng():
    e = _engine()
    yield e
    e.close()


def _residues(x, t=T):
    return np.mod(np.rint(x).astype(np.int64), t)


def _prepare(e, M, baby_steps=0, ntt_bytes=0):
    rows = [e.plain(r, 1.0) for r in M]
    d = e.diag_prepare(rows, baby_steps, ntt_bytes)
    e.dispose_many(rows)
    return d


def _banded(rng, R, dim, offsets):
    M = np.zeros((R, dim))
    for off in offsets:
        for r in range(R):
            if r + off < dim:
                M[r, r + off] = rng.integers(-4, 5)
    return M


def _group_sizes(M, n, n1, t=T):
    """Diagonals per giant-step group with a nonzero diagonal, in storage order (by g, then b, then h)."""
    nz = dg.diagonal_flags(_residues(M, t), n)
    return [int(c) for c in nz.reshape(2, n // 2 // n1, n1).sum(axis=(0, 2)) if c]


def _words(e, ys):
    return [y.export_raw(ch, 0) for y in ys for ch in range(e.P)]


def _lift(m, t, q):
    """multiply_plain's lift of a plaintext coefficient mod t into q: m >= (t + 1) / 2 becomes m + q - t."""
    m = np.asarray(m, np.uint64)
    return np.where(m >= (t + 1) // 2, m + np.uint64(q - t), m)


# ------------------------------------------------------------------------------------------------ resident words
@pytest.mark.parametrize("t,n", [(T, 4096), (549764251649, 8192), (957181001729, 16384)])
def test_resident_words_are_the_lifted_forward_transforms(t, n):
    from oracle.oracle_py import Oracle
    e = _engine(t, n)
    try:
        orc = Oracle(t, n, -1, 10, 20)
        assert orc.q == e.q
        rng = np.random.default_rng(n)
        half = n // 2
        # bands in the first row of slots (b = 0) and one reaching into the second row (b = 1); negative weights exercise the lift
        M = _banded(rng, 300, half + 700, [0, 5, 17, half + 300])
        d = _prepare(e, M, 16, ALL)
        info, ni = d.info(), d.ntt_info()
        assert ni["diags"] == info["n_diags"] and ni["giant_steps"] == len(_group_sizes(M, n, 16, t))
        seen_b = set()
        for j in range(info["n_diags"]):
            pl, (b, g, h) = d.export(0, j)
            seen_b.add(b)
            got = d.export_ntt(0, j)
            assert got.shape == (len(e.q), n)
            for l, q in enumerate(e.q):
                assert np.array_equal(got[l], orc.ntt(l, _lift(pl, t, q))), (j, l)
        assert seen_b == {0, 1}
        d.dispose()
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------ bit identity of the product
def _compare(e, M, n1, budget, xs):
    d0 = _prepare(e, M, n1, 0)
    d1 = _prepare(e, M, n1, budget)
    e.op_counts(reset=True)
    y0 = e.mat_mul_diagonal(d0, xs)
    c0 = e.op_counts(reset=True)
    y1 = e.mat_mul_diagonal(d1, xs)
    c1 = e.op_counts(reset=True)
    assert c0 == c1
    for a, b in zip(_words(e, y0), _words(e, y1)):
        assert np.array_equal(a, b)
    for y in y0 + y1:
        y.dispose()
    ni = d1.ntt_info()
    d0.dispose()
    d1.dispose()
    return ni


def _budgets(e, sizes):
    per = e.P * len(e.q) * e.N * 8
    assert sizes[1] >= 2
    return {"none": (0, 0), "one_group": (sizes[0] * per, 1), "mid_group": ((sizes[0] + 1) * per, 1),
            "all": (ALL, len(sizes))}


@pytest.mark.parametrize("B", [1, 3, 9])
@pytest.mark.parametrize("budget", ["none", "one_group", "mid_group", "all"])
def test_product_is_word_for_word_the_coefficient_forms(eng, budget, B):
    rng = np.random.default_rng(100 + B)
    R, dim, n1 = 37, 2100, 16
    M = rng.integers(-1, 2, (R, dim)).astype(np.float64)
    sizes = _group_sizes(M, N, n1)
    nb, groups = _budgets(eng, sizes)[budget]
    xs = [eng.encrypt(rng.integers(-3, 4, dim).astype(np.float64), 1.0) for _ in range(B)]
    ni = _compare(eng, M, n1, nb, xs)
    assert ni["giant_steps"] == groups and ni["diags"] == sum(sizes[:groups])


@pytest.mark.parametrize("B", [1, 2, 3, 5, 9])
def test_resident_mac(eng, B):
    """The MAC over the wholly resident matrix gives the coefficient form's words, for every client-count instantiation (B = 9: two
    passes of 8), with groups whose lengths are not multiples of the 8-term re-centring period."""
    rng = np.random.default_rng(200 + B)
    M = rng.integers(-1, 2, (37, 2100)).astype(np.float64) * (rng.random((37, 2100)) < 0.7)
    assert any(s % 8 for s in _group_sizes(M, N, 16))
    xs = [eng.encrypt(rng.integers(-3, 4, 2100).astype(np.float64), 1.0) for _ in range(B)]
    _compare(eng, M, 16, ALL, xs)


def test_resident_mac_option_refusals(eng):
    """diag_mac_resident, which once picked the resident MAC kernel, is an unknown option now, for the values it used to accept."""
    for old in (0, 2, 8):
        assert _code(lambda: eng.set_option("diag_mac_resident", old)) == ERR_INVALID
    rng = np.random.default_rng(81)
    M = rng.integers(-1, 2, (20, 100)).astype(np.float64)
    d = _prepare(eng, M, 0, ALL)
    v = rng.integers(-2, 3, 100).astype(np.float64)
    y = eng.mat_mul_diagonal(d, [eng.encrypt(v, 1.0)])[0]
    assert np.array_equal(eng.decrypt(y), M @ v)
    y.dispose()
    d.dispose()


def test_giant_steps_with_gaps(eng):
    """Nonzero diagonals in giant steps 0, 3 and 7 only (n1 = 16), partly and wholly resident."""
    rng = np.random.default_rng(21)
    M = _banded(rng, 500, 700, [0, 2, 3 * 16 + 1, 3 * 16 + 9, 7 * 16])
    sizes = _group_sizes(M, N, 16)
    assert sizes == [2, 2, 1]
    per = eng.P * len(eng.q) * N * 8
    xs = [eng.encrypt(rng.integers(-3, 4, 700).astype(np.float64), 1.0) for _ in range(2)]
    for nb, groups in ((4 * per, 2), (ALL, 3)):
        assert _compare(eng, M, 16, nb, xs)["giant_steps"] == groups


def test_two_key_slots_in_one_call():
    server = _engine(seed=100)
    client = _engine(seed=200)
    try:
        slot = server.add_client_compact(client.save_compact_keys(public=False))
        rng = np.random.default_rng(31)
        M = rng.integers(-1, 2, (300, 2500)).astype(np.float64) * (rng.random((300, 2500)) < 0.5)
        vals = [rng.integers(-2, 3, 2500).astype(np.float64) for _ in range(3)]
        xs = [server.encrypt(vals[0], 1.0)]
        for v in vals[1:]:
            xv = server.import_raw(client.encrypt(v, 1.0).export_raw(0, 0), 1, 2500, 1.0)
            xv.set_key_slot(slot)
            xs.append(xv)
        probe = _prepare(server, M)
        sizes = _group_sizes(M, N, probe.info()["n1"])
        probe.dispose()
        per = server.P * len(server.q) * N * 8
        d = _prepare(server, M, 0, (sizes[0] + sizes[1]) * per)
        ys = server.mat_mul_diagonal(d, xs)
        assert [y.key_slot for y in ys] == [0, slot, slot]
        assert np.array_equal(server.decrypt(ys[0]), M @ vals[0])
        for y, v in zip(ys[1:], vals[1:]):
            assert np.array_equal(client.decrypt(client.import_raw(y.export_raw(0, 0), 1, 300, 1.0)), M @ v)
        d.dispose()
        _compare(server, M, 0, (sizes[0] + sizes[1]) * per, xs)
    finally:
        client.close()
        server.close()


def test_integer_path():
    e = _engine(int_path=True)
    try:
        rng = np.random.default_rng(41)
        M = rng.integers(-1, 2, (500, 3100)).astype(np.float64) * (rng.random((500, 3100)) < 0.4)
        xs = [e.encrypt(rng.integers(-2, 3, 3100).astype(np.float64), 1.0) for _ in range(3)]
        sizes = _group_sizes(M, N, 16)
        per = e.P * len(e.q) * N * 8
        for nb in ((sizes[0] + 1) * per, ALL):
            _compare(e, M, 16, nb, xs)
    finally:
        e.close()


def test_ring_16384():
    e = _engine(957181001729, 16384)
    try:
        rng = np.random.default_rng(51)
        M = _banded(rng, 2000, 9000, [0, 1, 40, 300, 8192 + 7])
        sizes = _group_sizes(M, 16384, 16, 957181001729)
        per = e.P * len(e.q) * 16384 * 8
        xs = [e.encrypt(rng.integers(-3, 4, 9000).astype(np.float64), 1.0) for _ in range(2)]
        for nb in (sizes[0] * per, ALL):
            _compare(e, M, 16, nb, xs)
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------ info and refusals
def _code(fn):
    with pytest.raises(CnheError) as ei:
        fn()
    return ei.value.code


def test_info_reports_the_budget(eng):
    rng = np.random.default_rng(61)
    M = rng.integers(-1, 2, (37, 2100)).astype(np.float64)
    sizes = _group_sizes(M, N, 16)
    per = eng.P * len(eng.q) * N * 8
    for nb, groups in ((0, 0), (sizes[0] * per - 1, 0), (sizes[0] * per, 1), ((sizes[0] + sizes[1]) * per + per - 1, 2), (ALL, len(sizes)),
                       ((1 << 64) - 1, len(sizes))):
        d = _prepare(eng, M, 16, nb)
        info, ni = d.info(), d.ntt_info()
        nd = sum(sizes[:groups])
        assert ni == dict(giant_steps=groups, diags=nd, bytes=nd * per), nb
        assert info["n_diags"] == sum(sizes)
        assert info["device_bytes"] == info["n_diags"] * N * 8 * eng.P + ni["bytes"]
        d.dispose()


def test_refusals_leave_the_context_usable(eng):
    from cryptonets_b200.engine import _p
    rng = np.random.default_rng(71)
    M = rng.integers(-1, 2, (20, 100)).astype(np.float64)
    rows = [eng.plain(r, 1.0) for r in M]
    enc_row = eng.encrypt(M[0], 1.0)
    assert _code(lambda: eng.diag_prepare(rows[:5] + [enc_row], 0, ALL)) == ERR_INVALID
    assert _code(lambda: eng.diag_prepare(rows, 3, ALL)) == ERR_INVALID
    d = eng.diag_prepare(rows, 0, ALL)
    d0 = eng.diag_prepare(rows, 0, 0)
    nd = d.ntt_info()["diags"]
    assert nd == d.info()["n_diags"]
    assert _code(lambda: d.export_ntt(0, nd)) == ERR_INVALID
    assert _code(lambda: d.export_ntt(0, -1)) == ERR_INVALID
    assert _code(lambda: d.export_ntt(eng.P, 0)) == ERR_INVALID
    assert _code(lambda: d0.export_ntt(0, 0)) == ERR_INVALID
    small = np.zeros(len(eng.q) * N - 1, np.uint64)
    from cryptonets_b200.engine import check
    assert _code(lambda: check(eng.L.cnhe_diag_export_ntt(eng.h, d.h, 0, 0, _p(small), small.size))) == ERR_INVALID
    other = _engine(seed=5)
    try:
        assert _code(lambda: check(other.L.cnhe_diag_export_ntt(other.h, d.h, 0, 0, _p(small), len(eng.q) * N + 1))) == ERR_INVALID
    finally:
        other.close()
    v = rng.integers(-2, 3, 100).astype(np.float64)
    y = eng.mat_mul_diagonal(d, [eng.encrypt(v, 1.0)])[0]
    assert np.array_equal(eng.decrypt(y), M @ v)
    d.dispose()
    d0.dispose()
    eng.dispose_many(rows + [enc_row])


# ------------------------------------------------------------------------------------------------ networks
def _chain(net):
    out, p = [], net
    while p is not None and hasattr(p, "Source"):
        out.append(p)
        p = p.Source
    return out[::-1]


@pytest.mark.parametrize("name", ["lola_large", "lola_cifar"])
def test_networks_with_a_partial_budget(name):
    """dense4 with 3 GiB of its diagonals in NTT form: from the same input ciphertexts the scores are word for word those of the
    coefficient-form matrix, and decrypt to the Raw backend's."""
    from cryptonets_b200 import networks as nw
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.raw import RawFactory
    build = getattr(nw, name)
    primes, k, imgs = ((nw.LOLA_LARGE_PRIMES, 7, nw.synthetic_mnist(1, seed=3)) if name == "lola_large" else
                       (nw.CIFAR_PRIMES, 8, nw.synthetic_cifar(1)))
    f = B200BfvFactory(primes, 16384, DecompositionBitCount=60, GaloisDecompositionBitCount=60, SmallModulusCount=k + 1, seed=5)
    try:
        coef, rd = build(f, imgs, dense_method="diagonal")
        coef.PrepareNetwork()
        ntt, _ = build(f, imgs, dense_method="diagonal", diag_ntt_bytes=3 << 30)
        ntt.PrepareNetwork()
        lc, ln = _chain(coef), _chain(ntt)
        ni = ln[5].DiagonalMatrix.NttInfo()
        assert 0 < ni["diags"] < ln[5].DiagonalMatrix.Info()["n_diags"] and ni["bytes"] <= 3 << 30
        m = rd.GetNext()
        for L in lc[1:5]:
            m = L.Apply(m)
        outs = []
        for chain in (lc, ln):
            y = m
            for L in chain[5:]:
                y = L.Apply(y)
            outs.append(y)
        eng = f.engine
        for a, b in zip(outs[0].vectors, outs[1].vectors):
            for ch in range(eng.P):
                for blk in range(a.vec.blocks):
                    assert np.array_equal(a.vec.export_raw(ch, blk), b.vec.export_raw(ch, blk))
        raw_net, _ = build(RawFactory(16384), imgs)
        raw_net.PrepareNetwork()
        got = np.asarray(outs[1].Decrypt()).reshape(-1)
        want = np.asarray(raw_net.GetNext().Decrypt()).reshape(-1)
        assert np.allclose(got, want, rtol=1e-9, atol=1e-9) and got.argmax() == want.argmax()
    finally:
        f.Dispose()
