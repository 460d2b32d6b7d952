"""The diagonal (baby-step / giant-step) matrix-vector product, cnhe_diag_prepare / cnhe_mat_mul_diagonal: bit for bit against the same
composition of the CPU oracle's encode, rotations, multiply_plain and add; decryption against M v mod t; several clients in one call; the
integer fallback; the refusals; and LoLa-Large / LoLa-CIFAR with their big dense layer on the diagonal method."""
import os

import numpy as np
import pytest

from cryptonets_b200 import diagonal as dg
from cryptonets_b200._lib import CnheError

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -3
T, N = 40961, 4096  # IFactory.cs:247-253's first prime, N = 4096, default coefficient modulus


def _engine(int_path=False, seed=1234):
    from cryptonets_b200.engine import Engine
    saved = os.environ.pop("CNHE_NTT_INT", None)
    if int_path:
        os.environ["CNHE_NTT_INT"] = "1"
    try:
        eng = Engine([T], N, 10, 20, -1)
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


def _small_matrix(rng, R, dim, density=1.0):
    M = rng.integers(-1, 2, (R, dim)).astype(np.float64)
    if density < 1.0:
        M *= rng.random((R, dim)) < density
    return M


def _residues(x, t=T):
    return np.mod(np.rint(x).astype(np.int64), t)


def _prepare(e, M, baby_steps=0, scale=1.0):
    rows = [e.plain(r, scale) for r in M]
    d = e.diag_prepare(rows, baby_steps)
    e.dispose_many(rows)
    return d


def test_bit_identical_to_the_oracle_composition(eng):
    """The exported diagonals are the oracle's encodings of the model's pre-rotated diagonals, and the output ciphertext is the oracle's
    rotate_columns, rotate_rows, multiply_plain, add composition in the same order, word for word."""
    from oracle.oracle_py import Oracle
    orc = Oracle(T, N, -1, 10, 20)
    assert orc.q == eng.q
    orc.keygen(1234)
    rng = np.random.default_rng(1)
    R, dim, n1 = 37, 2100, 16
    M = _small_matrix(rng, R, dim)
    v = rng.integers(-3, 4, dim).astype(np.float64)
    d = _prepare(eng, M, n1)
    info = d.info()
    assert (info["n_rows"], info["dim"], info["n1"], info["n2"]) == (R, dim, n1, N // 2 // n1)
    model = dg.prerotated_diagonals(_residues(M), N, n1, T)
    assert info["n_diags"] == len(model)
    assert info["device_bytes"] == info["n_diags"] * N * 8
    x = eng.encrypt(v, 1.0)
    ct = x.export_raw(0, 0)
    kv = orc.rotate_columns(ct)
    baby = {}
    inner = {}
    for j in range(info["n_diags"]):
        pl, (b, g, h) = d.export(0, j)
        assert np.array_equal(pl, orc.encode(model[(b, g, h)].astype(np.uint64))), (b, g, h)
        if (b, h) not in baby:
            src = kv if b else ct
            baby[(b, h)] = orc.rotate_rows(src, h) if h else src
        term = orc.multiply_plain(baby[(b, h)], pl)
        inner[g] = term if g not in inner else orc.add(inner[g], term)
    want = None
    for g in sorted(inner):
        r = orc.rotate_rows(inner[g], n1 * g) if g else inner[g]
        want = r if want is None else orc.add(want, r)
    y = eng.mat_mul_diagonal(d, [x])[0]
    assert np.array_equal(y.export_raw(0, 0), want)
    assert np.array_equal(_residues(eng.decrypt(y)), np.mod(_residues(M).astype(object) @ _residues(v).astype(object), T).astype(np.int64))
    d.dispose()


@pytest.mark.parametrize("R", [1, N // 2 - 1, N // 2 + 3, N])
def test_decrypts_to_the_matrix_vector_product(eng, R):
    rng = np.random.default_rng(R)
    dim = 3000  # crosses into the second row of slots
    M = _small_matrix(rng, R, dim, density=0.3)
    v = rng.integers(-1, 2, dim).astype(np.float64)
    d = _prepare(eng, M, scale=2.0)
    nz = dg.diagonal_flags(_residues(2 * M), N)
    info = d.info()
    assert info["n1"] == dg.plan_baby_steps(nz, N, eng.galois_elts())[0]
    assert info["n_diags"] == int(nz.sum())
    x = eng.encrypt(v, 3.0)
    y = eng.mat_mul_diagonal(d, [x])[0]
    assert (y.dim, y.scale) == (R, 6.0)
    assert np.array_equal(eng.decrypt(y), M @ v)
    d.dispose()


def test_banded_matrix_and_the_row_path(eng):
    """A banded matrix keeps only its nonzero diagonals, and decrypts to what the row-major product with ForceDenseFormat decrypts to."""
    rng = np.random.default_rng(7)
    R = dim = 200
    M = np.zeros((R, dim))
    for off in (0, 1, 5, 17):
        for r in range(R):
            if r + off < dim:
                M[r, r + off] = rng.integers(-4, 5)
    v = rng.integers(-3, 4, dim).astype(np.float64)
    d = _prepare(eng, M)
    nz = dg.diagonal_flags(_residues(M), N)
    assert d.info()["n_diags"] == int(nz.sum()) == 4  # one diagonal per band: 200 rows and columns sit in the first row of slots
    x = eng.encrypt(v, 1.0)
    y = eng.mat_mul_diagonal(d, [x])[0]
    rows = [eng.plain(r, 1.0) for r in M]
    ref = eng.mat_mul_rowmajor(rows, x, force_dense=True)
    assert np.array_equal(eng.decrypt(y), eng.decrypt(ref))
    assert np.array_equal(eng.decrypt(y), M @ v)
    d.dispose()


def test_several_clients_in_one_call():
    """Three inputs of three key slots in one call: each output is bit-identical to its own single-vector call and decrypts under its
    client's key."""
    server = _engine(seed=100)
    clients = [_engine(seed=200 + j) for j in range(2)]
    try:
        slots = [0] + [server.add_client_compact(c.save_compact_keys(public=False)) for c in clients]
        rng = np.random.default_rng(11)
        M = _small_matrix(rng, 300, 2500, density=0.5)
        vals = [rng.integers(-2, 3, 2500).astype(np.float64) for _ in range(3)]
        xs = [server.encrypt(vals[0], 1.0)]
        for j, c in enumerate(clients):
            cv = c.encrypt(vals[j + 1], 1.0)
            xv = server.import_raw(cv.export_raw(0, 0), 1, 2500, 1.0)
            xv.set_key_slot(slots[j + 1])
            xs.append(xv)
        d = _prepare(server, M)
        together = server.mat_mul_diagonal(d, xs)
        for j in range(3):
            alone = server.mat_mul_diagonal(d, [xs[j]])[0]
            assert together[j].key_slot == slots[j]
            assert np.array_equal(together[j].export_raw(0, 0), alone.export_raw(0, 0)), j
            owner = server if j == 0 else clients[j - 1]
            got = owner.decrypt(owner.import_raw(together[j].export_raw(0, 0), 1, 300, 1.0)) if j else server.decrypt(together[j])
            assert np.array_equal(got, M @ vals[j]), j
        d.dispose()
    finally:
        for c in clients:
            c.close()
        server.close()


def test_integer_fallback_gives_the_same_ciphertexts():
    rng = np.random.default_rng(13)
    M = _small_matrix(rng, 500, 3100, density=0.4)
    v = rng.integers(-2, 3, 3100).astype(np.float64)
    outs = []
    for int_path in (False, True):
        e = _engine(int_path)
        try:
            d = _prepare(e, M)
            x = e.encrypt(v, 1.0)
            outs.append((d.export(0, 3)[0], e.mat_mul_diagonal(d, [x])[0].export_raw(0, 0)))
            d.dispose()
        finally:
            e.close()
    assert np.array_equal(outs[0][0], outs[1][0])
    assert np.array_equal(outs[0][1], outs[1][1])


def _code(fn):
    with pytest.raises(CnheError) as ei:
        fn()
    return ei.value.code


def test_refusals_leave_the_context_usable(eng):
    rng = np.random.default_rng(17)
    M = _small_matrix(rng, 20, 100)
    rows = [eng.plain(r, 1.0) for r in M]
    enc_row = eng.encrypt(M[0], 1.0)
    sparse_row = eng.plain(M[0], 1.0, fmt=1)
    long_row = eng.plain(np.ones(N + 10), 1.0)
    short_row = eng.plain(M[0][:50], 1.0)
    other_scale = eng.plain(M[0], 2.0)
    assert _code(lambda: eng.diag_prepare(rows[:5] + [enc_row])) == ERR_INVALID
    assert _code(lambda: eng.diag_prepare(rows[:5] + [sparse_row])) == ERR_INVALID
    assert _code(lambda: eng.diag_prepare([long_row])) == ERR_INVALID
    assert _code(lambda: eng.diag_prepare(rows[:5] + [short_row])) == ERR_INVALID
    assert _code(lambda: eng.diag_prepare(rows[:5] + [other_scale])) == ERR_INVALID
    assert _code(lambda: eng.diag_prepare(rows[:1] * (N + 1))) == ERR_INVALID
    assert _code(lambda: eng.diag_prepare(rows, baby_steps=3)) == ERR_INVALID
    assert _code(lambda: eng.diag_prepare(rows, baby_steps=N)) == ERR_INVALID
    d = eng.diag_prepare(rows)
    v = rng.integers(-2, 3, 100).astype(np.float64)
    assert _code(lambda: eng.mat_mul_diagonal(d, [eng.encrypt(v[:90], 1.0)])) == ERR_INVALID
    assert _code(lambda: eng.mat_mul_diagonal(d, [eng.plain(v, 1.0)])) == ERR_INVALID
    assert _code(lambda: eng.mat_mul_diagonal(d, [eng.encrypt(np.ones(N + 10), 1.0)])) == ERR_INVALID
    # a client without Galois keys: the rotations cannot run
    c = _engine(seed=300)
    try:
        slot = eng.add_client_compact(c.save_compact_keys(public=False, galois=[]))
        xv = eng.import_raw(c.encrypt(v, 1.0).export_raw(0, 0), 1, 100, 1.0)
        xv.set_key_slot(slot)
        assert _code(lambda: eng.mat_mul_diagonal(d, [xv])) == ERR_STATE
        eng.remove_client(slot)
    finally:
        c.close()
    y = eng.mat_mul_diagonal(d, [eng.encrypt(v, 1.0)])[0]
    assert np.array_equal(eng.decrypt(y), M @ v)
    d.dispose()
    eng.dispose_many(rows + [enc_row, sparse_row, long_row, short_row, other_scale])


# ------------------------------------------------------------------------------------------------ networks
def _chain(net):
    out, p = [], net
    while p is not None and hasattr(p, "Source"):
        out.append(p)
        p = p.Source
    return out[::-1]


def _budget_into_last_layer(f, net, rd):
    m = rd.GetNext()
    for layer in _chain(net)[1:-1]:
        m = layer.Apply(m)
    b = min(f.engine.noise_budget(v.vec, ch, 0) for v in m.vectors for ch in range(f.engine.P))
    m.Dispose()
    return b


@pytest.mark.parametrize("extra_prime", [1, 0])
@pytest.mark.parametrize("name", ["lola_large", "lola_cifar"])
def test_networks_on_the_diagonal_method(name, extra_prime):
    """Scores equal the Raw backend's at one coefficient prime more than the reference's SmallModulusCount (7 for LoLa-Large, 8 for
    LoLa-CIFAR), where the budget entering the last layer is also higher than on the row path, and at the reference's own count, where
    the row path does not decrypt (DESIGN.md section 7.1)."""
    from cryptonets_b200 import networks as nw
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.raw import RawFactory
    build = getattr(nw, name)
    primes, k, imgs = ((nw.LOLA_LARGE_PRIMES, 7, nw.synthetic_mnist(1, seed=3)) if name == "lola_large" else
                       (nw.CIFAR_PRIMES, 8, nw.synthetic_cifar(1)))
    f = B200BfvFactory(primes, 16384, DecompositionBitCount=60, GaloisDecompositionBitCount=60, SmallModulusCount=k + extra_prime, seed=5)
    try:
        net, _ = build(f, imgs, dense_method="diagonal")
        net.PrepareNetwork()
        raw_net, _ = build(RawFactory(16384), imgs)
        raw_net.PrepareNetwork()
        got = np.asarray(net.GetNext().Decrypt()).reshape(-1)
        want = np.asarray(raw_net.GetNext().Decrypt()).reshape(-1)
        assert np.allclose(got, want, rtol=1e-9, atol=1e-9) and got.argmax() == want.argmax()
        if not extra_prime:
            return
        budgets = {}
        for method in ("rows", "diagonal"):
            n2, rd2 = build(f, imgs, dense_method=method)
            n2.PrepareNetwork()
            budgets[method] = _budget_into_last_layer(f, n2, rd2)
            n2.DisposeNetwork()
        assert budgets["diagonal"] > budgets["rows"], budgets
    finally:
        f.Dispose()
