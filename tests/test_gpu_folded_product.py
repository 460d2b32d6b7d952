"""The folded diagonal product for matrices with few rows, cnhe_diag_prepare_folded / cnhe_mat_mul_diagonal: bit for bit against the
CPU oracle's composition (encode, rotations, multiply_plain, add, rotate_columns, the fold hops and the mask) at N = 4096, 8192 and
16384, with resident and streamed diagonals, 53/56-bit moduli and the integer path; padding slots decrypt to 0; several clients in one
call; operation counts; the refusals; and lola_small, LoLa-CIFAR and LoLa-Large with a folded score layer against the Raw backend."""
import numpy as np
import pytest

from cryptonets_b200 import diagonal as dg
from cryptonets_b200._lib import CnheError
from test_poly4_constants import _is_prime

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -3


def _prime(bits, N):
    c = ((1 << bits) - 1) // (2 * N) * (2 * N) + 1
    while not _is_prime(c):
        c -= 2 * N
    return c


# name: plain prime, N, decomposition bit count, coefficient moduli (None: the default), environment at context creation
CONTEXTS = {
    "n4096": dict(t=40961, N=4096, dbc=10, q=None, env={}),
    "n8192": dict(t=2277377, N=8192, dbc=40, q=None, env={}),
    "n16384": dict(t=786433, N=16384, dbc=60, q=None, env={}),
    "n4096-q53": dict(t=40961, N=4096, dbc=10, q=[_prime(53, 4096), _prime(56, 4096)], env={}),
    "n8192-int": dict(t=2277377, N=8192, dbc=40, q=None, env={"CNHE_NTT_INT": "1"}),
}


def _pair(name, monkeypatch, seed=31):
    from cryptonets_b200.engine import Engine
    from oracle.oracle_py import Oracle
    cfg = CONTEXTS[name]
    monkeypatch.delenv("CNHE_NTT_INT", raising=False)
    for var, v in cfg["env"].items():
        monkeypatch.setenv(var, v)
    eng = Engine([cfg["t"]], cfg["N"], cfg["dbc"], 20, -1, coeff_moduli=cfg["q"])
    for var in cfg["env"]:
        monkeypatch.delenv(var, raising=False)
    eng.keygen(seed)
    orc = Oracle(cfg["t"], cfg["N"], -1, cfg["dbc"], 20, custom_q=cfg["q"])
    orc.keygen(seed)
    return eng, orc


def _residues(x, t):
    return np.mod(np.rint(x).astype(np.int64), t)


def _prepare(e, M, fold_width=0, baby_steps=0, ntt_bytes=0, scale=1.0):
    rows = [e.plain(r, scale) for r in M]
    d = e.diag_prepare(rows, baby_steps, ntt_bytes, fold_width=fold_width)
    e.dispose_many(rows)
    return d


def _oracle_product(orc, d, ct, N, dim, R):
    """The folded product as the oracle's composition, in the library's order of operations."""
    info = d.info()
    n1, W, half = info["n1"], d.fold_width(), N // 2
    baby, inner = {}, {}
    for j in range(info["n_diags"]):
        pl, (b, g, h) = d.export(0, j)
        assert b == 0
        if h not in baby:
            baby[h] = orc.rotate_rows(ct, h) if h else ct
        term = orc.multiply_plain(baby[h], pl)
        inner[g] = term if g not in inner else orc.add(inner[g], term)
    y = None
    for g in sorted(inner):
        r = orc.rotate_rows(inner[g], n1 * g) if g else inner[g]
        y = r if y is None else orc.add(y, r)
    if dim > half:
        y = orc.add(y, orc.rotate_columns(y))
    s = W
    while s < half:
        y = orc.add(y, orc.rotate_rows(y, -s))
        s *= 2
    mask = np.zeros(N, np.uint64)
    mask[:R] = 1
    return orc.multiply_plain(y, orc.encode(mask))


# (context, R, dim, fold width or 0, resident): N = 4096 with dim > N/2 runs the column fold
CASES = [("n4096", 10, 3000, 0, False), ("n4096", 10, 3000, 0, True), ("n4096", 7, 1500, 64, False), ("n8192", 10, 845, 0, False),
         ("n8192", 10, 845, 0, True), ("n16384", 10, 5488, 0, True), ("n16384", 13, 9000, 32, False), ("n4096-q53", 10, 3000, 0, True),
         ("n4096-q53", 5, 1200, 0, False), ("n8192-int", 10, 845, 0, False), ("n8192-int", 10, 845, 0, True)]


@pytest.mark.parametrize("name,R,dim,W,resident", CASES)
def test_bit_identical_to_the_oracle_composition(name, R, dim, W, resident, monkeypatch):
    eng, orc = _pair(name, monkeypatch)
    try:
        N, t = eng.N, CONTEXTS[name]["t"]
        assert orc.q == eng.q
        rng = np.random.default_rng(R * dim)
        M = rng.integers(-4, 5, (R, dim)).astype(np.float64)
        v = rng.integers(-9, 10, dim).astype(np.float64)
        d = _prepare(eng, M, W, ntt_bytes=None if resident else 0)
        info = d.info()
        plan = dg.plan_folded(_residues(M, t), N, eng.galois_elts(), W)
        assert (d.fold_width(), info["n1"], info["n2"]) == (plan[0], plan[1], plan[0] // plan[1])
        model = dg.folded_diagonals(_residues(M, t), N, plan[0], plan[1], t)
        assert info["n_diags"] == len(model) and (info["n_rows"], info["dim"]) == (R, dim)
        for j in range(info["n_diags"]):
            pl, bgh = d.export(0, j)
            assert np.array_equal(pl, orc.encode(model[bgh].astype(np.uint64))), bgh
        nt = d.ntt_info()
        assert nt["diags"] == (info["n_diags"] if resident else 0)
        x = eng.encrypt(v, 1.0)
        y = eng.mat_mul_diagonal(d, [x])[0]
        assert (y.dim, y.blocks) == (R, 1)
        want = _oracle_product(orc, d, x.export_raw(0, 0), N, dim, R)
        assert np.array_equal(y.export_raw(0, 0), want)
        assert np.array_equal(_residues(eng.decrypt(y), t), _residues(M @ v, t))
        full = eng.decrypt(eng.import_raw(y.export_raw(0, 0), 1, N, 1.0))  # every slot: the padding decrypts to 0
        assert np.array_equal(_residues(full[:R], t), _residues(M @ v, t)) and not _residues(full[R:], t).any()
        d.dispose()
    finally:
        eng.close()


def test_several_clients_in_one_call(monkeypatch):
    """B = 1, 3 and 9 inputs of two key slots in one call: each output is bit-identical to its own single-vector call."""
    from cryptonets_b200.engine import Engine
    server, _ = _pair("n4096", monkeypatch, seed=100)
    client = Engine([CONTEXTS["n4096"]["t"]], 4096, 10, 20, -1)
    client.keygen(200)
    try:
        slot = server.add_client_compact(client.save_compact_keys(public=False))
        rng = np.random.default_rng(3)
        R, dim = 10, 2500
        M = rng.integers(-3, 4, (R, dim)).astype(np.float64)
        d = _prepare(server, M, ntt_bytes=None)
        vals = [rng.integers(-5, 6, dim).astype(np.float64) for _ in range(9)]
        xs = []
        for j, v in enumerate(vals):
            if j % 2:
                xv = server.import_raw(client.encrypt(v, 1.0).export_raw(0, 0), 1, dim, 1.0)
                xv.set_key_slot(slot)
            else:
                xv = server.encrypt(v, 1.0)
            xs.append(xv)
        alone = [server.mat_mul_diagonal(d, [x])[0].export_raw(0, 0) for x in xs]
        for B in (1, 3, 9):
            together = server.mat_mul_diagonal(d, xs[:B])
            for j in range(B):
                assert together[j].key_slot == (slot if j % 2 else 0)
                assert np.array_equal(together[j].export_raw(0, 0), alone[j]), (B, j)
        for j in (0, 1):
            owner = client if j % 2 else server
            got = owner.decrypt(owner.import_raw(alone[j], 1, R, 1.0))
            assert np.array_equal(got, M @ vals[j]), j
        d.dispose()
    finally:
        client.close()
        server.close()


@pytest.mark.parametrize("dim", [845, 3000])
def test_operation_counts(dim, monkeypatch):
    eng, _ = _pair("n4096", monkeypatch)
    try:
        N, half, t, B, R = eng.N, eng.N // 2, CONTEXTS["n4096"]["t"], 3, 10
        rng = np.random.default_rng(dim)
        M = rng.integers(-3, 4, (R, dim)).astype(np.float64)
        d = _prepare(eng, M)
        info, W = d.info(), d.fold_width()
        n1, nd = info["n1"], info["n_diags"]
        keys = dg.folded_diagonals(_residues(M, t), N, W, n1, t).keys()
        hops = dg.rotation_hops(N, eng.galois_elts())
        babies, giants = {h for _, _, h in keys}, {g for _, g, _ in keys}
        folds = half.bit_length() - W.bit_length()
        col = 1 if dim > half else 0
        xs = [eng.encrypt(rng.integers(-3, 4, dim).astype(np.float64), 1.0) for _ in range(B)]
        eng.op_counts(reset=True)
        eng.mat_mul_diagonal(d, xs)
        got = eng.op_counts(reset=True)
        rot = sum(hops[h] for h in babies if h) + sum(hops[n1 * g] for g in giants if g) + folds
        assert got["Rotation"] == B * rot and got["ColumnRotation"] == B * col, got
        assert rot + col == dg.plan_folded(_residues(M, t), N, eng.galois_elts())[2]
        assert got["PlainMultiplication"] == B * (nd + 1), got
        assert got["Addition"] == B * (nd - len(giants) + folds + col), got
        assert got["AddMany"] == (B if len(giants) > 1 else 0), got
        d.dispose()
    finally:
        eng.close()


def _code(fn):
    with pytest.raises(CnheError) as ei:
        fn()
    return ei.value.code


def test_refusals_leave_the_context_usable(monkeypatch):
    eng, _ = _pair("n4096", monkeypatch)
    try:
        N = eng.N
        rng = np.random.default_rng(17)
        M = rng.integers(-2, 3, (20, 100)).astype(np.float64)
        rows = [eng.plain(r, 1.0) for r in M]
        enc_row = eng.encrypt(M[0], 1.0)
        long_row = eng.plain(np.ones(N + 10), 1.0)
        other_scale = eng.plain(M[0], 2.0)
        fold = lambda rs, **kw: eng.diag_prepare(rs, kw.pop("baby_steps", 0), fold_width=kw.pop("fold_width", 0))
        assert _code(lambda: fold(rows[:1] * (N // 2 + 1))) == ERR_INVALID          # more than N/2 rows
        assert _code(lambda: fold(rows, fold_width=24)) == ERR_INVALID               # not a power of two
        assert _code(lambda: fold(rows, fold_width=16)) == ERR_INVALID               # below the row count
        assert _code(lambda: fold(rows, fold_width=N)) == ERR_INVALID                # above N/2
        assert _code(lambda: fold(rows, fold_width=-1)) == ERR_INVALID
        assert _code(lambda: fold(rows, fold_width=32, baby_steps=64)) == ERR_INVALID  # n1 does not divide W
        assert _code(lambda: fold(rows, baby_steps=3)) == ERR_INVALID
        assert _code(lambda: fold([long_row])) == ERR_INVALID                         # more than N columns
        assert _code(lambda: fold(rows[:5] + [enc_row])) == ERR_INVALID
        assert _code(lambda: fold(rows[:5] + [other_scale])) == ERR_INVALID
        d = fold(rows, fold_width=32, baby_steps=8)
        assert (d.fold_width(), d.info()["n1"], d.info()["n2"]) == (32, 8, 4)
        v = rng.integers(-2, 3, 100).astype(np.float64)
        assert _code(lambda: eng.mat_mul_diagonal(d, [eng.encrypt(v[:90], 1.0)])) == ERR_INVALID
        assert _code(lambda: eng.mat_mul_diagonal(d, [eng.plain(v, 1.0)])) == ERR_INVALID
        from cryptonets_b200.engine import Engine
        c = Engine([CONTEXTS["n4096"]["t"]], N, 10, 20, -1)
        c.keygen(300)
        try:  # a client without Galois keys: the rotations cannot run
            slot = eng.add_client_compact(c.save_compact_keys(public=False, galois=[]))
            xv = eng.import_raw(c.encrypt(v, 1.0).export_raw(0, 0), 1, 100, 1.0)
            xv.set_key_slot(slot)
            assert _code(lambda: eng.mat_mul_diagonal(d, [xv])) == ERR_STATE
            eng.remove_client(slot)
        finally:
            c.close()
        y = eng.mat_mul_diagonal(d, [eng.encrypt(v, 1.0)])[0]
        assert np.array_equal(eng.decrypt(y), M @ v)
        unfolded = eng.diag_prepare(rows)
        assert unfolded.fold_width() == 0
        unfolded.dispose()
        d.dispose()
        eng.dispose_many(rows + [enc_row, long_row, other_scale])
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ networks
def _score_budget(f, m):
    return min(f.engine.noise_budget(v.vec, ch, b) for v in m.vectors for ch in range(f.engine.P) for b in range(v.vec.blocks))


@pytest.mark.parametrize("name", ["lola_small", "lola_cifar", "lola_large"])
def test_networks_with_a_folded_score_layer(name):
    """Scores equal the Raw backend's at one coefficient prime more than the reference's SmallModulusCount; the noise budget left at the
    scores is printed for the rows and the folded score layer."""
    from cryptonets_b200 import networks as nw
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.raw import RawFactory
    build = getattr(nw, name)
    if name == "lola_small":
        f = B200BfvFactory(nw.LOLA_SMALL_PRIMES, 8192, DecompositionBitCount=40, GaloisDecompositionBitCount=40, SmallModulusCount=4, seed=5)
        imgs, N, kw = nw.synthetic_mnist(2, seed=6), 8192, lambda m: dict(dense_method=m)
    else:
        primes, k, imgs = ((nw.LOLA_LARGE_PRIMES, 7, nw.synthetic_mnist(1, seed=3)) if name == "lola_large" else
                           (nw.CIFAR_PRIMES, 8, nw.synthetic_cifar(1)))
        f = B200BfvFactory(primes, 16384, DecompositionBitCount=60, GaloisDecompositionBitCount=60, SmallModulusCount=k + 1, seed=5)
        N, kw = 16384, lambda m: dict(dense_method="diagonal", score_method=m)
    try:
        budgets = {}
        for method in ("folded", "rows"):
            net, _ = build(f, imgs, **kw(method))
            net.PrepareNetwork()
            raw_net, _ = build(RawFactory(N), imgs)
            raw_net.PrepareNetwork()
            for _ in range(len(imgs)):
                m = net.GetNext()
                budgets.setdefault(method, []).append(_score_budget(f, m))
                got = np.asarray(m.Decrypt()).reshape(-1)
                want = np.asarray(raw_net.GetNext().Decrypt()).reshape(-1)
                assert np.allclose(got, want, rtol=1e-9, atol=1e-9) and got.argmax() == want.argmax(), method
                if method == "folded":
                    assert m.vectors[0].vec.blocks == 1 and m.vectors[0].vec.dim == 10
                m.Dispose()
            net.DisposeNetwork()
        print("%s: noise budget at the scores, rows %s bits, folded %s bits" % (name, budgets["rows"], budgets["folded"]))
        assert min(budgets["folded"]) > 0
    finally:
        f.Dispose()
