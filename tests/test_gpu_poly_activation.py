"""cnhe_layer_poly2: the quadratic activation A x^2 + B x + C with the three terms applied in the BEHZ floor kernel.

Every output word must equal the CPU oracle's composition relinearize(multiply_plain(multiply(x, x), A)) + multiply_plain(x, B) +
add_plain(C), per plaintext prime (a term that is 0 mod the prime is skipped there), on every path the product takes: fused square or
separate kernels, fused or digit key switch, the FP64 and the integer floor, N = 4096 / 8192 / 16384 and moduli of 50 bits and more.
(1, 0, 0) is the square's layer word for word, mixed key slots give each client's words, and two networks with their squares replaced
decrypt to the Raw backend."""
import numpy as np
import pytest

from cryptonets_b200._lib import CnheError

pytestmark = pytest.mark.gpu

ERR_INVALID = -1


def _is_prime(n):
    if n < 2:
        return False
    for sp in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):
        if n % sp == 0:
            return n == sp
    d, s = n - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    for a in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):
        x = pow(a, d, n)
        if x in (1, n - 1):
            continue
        for _ in range(s - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def _prime(bits, N):
    c = ((1 << bits) - 1) // (2 * N) * (2 * N) + 1
    while not _is_prime(c):
        c -= 2 * N
    return c


# name: plain primes, N, decomposition bit count, coefficient moduli (None: the default), environment at context creation (CNHE_NTT_INT:
# the integer floor k_behz_floor)
CONTEXTS = {
    "n4096": dict(t=[40961], N=4096, dbc=10, q=None, env={}),
    "n8192-cryptonets": dict(t=[549764251649, 549764284417], N=8192, dbc=10, q=None, env={}),
    "n16384": dict(t=[786433], N=16384, dbc=60, q=None, env={}),
    "n8192-int": dict(t=[2277377, 2424833], N=8192, dbc=40, q=None, env={"CNHE_NTT_INT": "1"}),
    "n4096-q53": dict(t=[40961], N=4096, dbc=10, q=[_prime(53, 4096), _prime(56, 4096)], env={}),
}


def _pair(name, monkeypatch):
    from cryptonets_b200.engine import Engine
    from oracle.oracle_py import Oracle
    cfg = CONTEXTS[name]
    monkeypatch.delenv("CNHE_NTT_INT", raising=False)
    for var, v in cfg["env"].items():
        monkeypatch.setenv(var, v)
    eng = Engine(cfg["t"], cfg["N"], cfg["dbc"], 20, -1, coeff_moduli=cfg["q"])
    for var in cfg["env"]:
        monkeypatch.delenv(var, raising=False)
    eng.keygen(31)
    orcs = []
    for ch, t in enumerate(cfg["t"]):
        o = Oracle(t, cfg["N"], -1, cfg["dbc"], 20, custom_q=cfg["q"])
        o.keygen(31 + ch)
        orcs.append(o)
    return eng, orcs


def _inputs(eng, n, seed, bound=200, dims=None):
    """n dense vectors of N slots each, or of the given dims (a dim that is not a multiple of N leaves padding slots in the last block)"""
    from cryptonets_b200.engine import DENSE
    rng = np.random.default_rng(seed)
    vals = [rng.integers(-bound, bound, d).astype(np.float64) for d in (dims or [eng.N] * n)]
    return vals, [eng.encrypt(v, 1.0, DENSE) for v in vals]


def _coeffs(eng, A, B, C):
    from cryptonets_b200.engine import SPARSE
    mk = lambda v: None if v is None else eng.plain(np.array([float(v)]), 1.0, SPARSE)
    return mk(A), mk(B), mk(C)


def _oracle_words(orc, x, A, B, C, fill=None):
    """relin(A . x^2) + B . x + C on the oracle, one plaintext prime; A, B, C integers (None = absent), reduced mod t here.  fill: None, C
    is the constant plaintext (every slot); else C is added to the first `fill` slots only (a dense vector's partly filled last block)"""
    t = orc.t
    A, B, C = (None if v is None or v % t == 0 else v % t for v in (A, B, C))
    out = orc.relinearize(orc.multiply_plain(orc.multiply(x, x), [A])) if A is not None else np.zeros(orc.ct_words, np.uint64)
    if B is not None:
        out = orc.add(out, orc.multiply_plain(x, [B]))
    if C is not None:
        out = orc.add_plain(out, [C] if fill is None else orc.encode(np.where(np.arange(orc.N) < fill, C, 0).astype(np.uint64)))
    return out


def _check_words(eng, orcs, xs, outs, A, B, C):
    for ch, orc in enumerate(orcs):
        for x, o in zip(xs, outs):
            assert o.blocks == x.blocks and o.dim == x.dim
            for bl in range(x.blocks):
                fill = x.dim % eng.N if bl == x.blocks - 1 and x.dim % eng.N else None
                assert np.array_equal(o.export_raw(ch, bl), _oracle_words(orc, x.export_raw(ch, bl), A, B, C, fill)), (ch, bl)


PATHS = [dict(CNHE_MUL_FUSED="1", CNHE_KS_FUSED="1"), dict(CNHE_MUL_FUSED="0", CNHE_KS_FUSED="0"), dict(CNHE_MUL_FUSED="1", CNHE_KS_FUSED="0"),
         dict(CNHE_MUL_FUSED="0", CNHE_KS_FUSED="1")]


@pytest.mark.parametrize("name", list(CONTEXTS))
def test_words_equal_oracle_composition(name, monkeypatch):
    eng, orcs = _pair(name, monkeypatch)
    try:
        _, xs = _inputs(eng, 4, 1, dims=[eng.N, eng.N // 2 + 3, eng.N, eng.N + 5])  # two with padding slots
        ts = CONTEXTS[name]["t"]
        # C in the upper half of t, negative B; then negative A and C with B absent
        cases = [(3, -7, ts[0] // 2 + 5), (-2, None, -11)]
        paths = PATHS if eng.N <= 8192 and not CONTEXTS[name]["env"] and CONTEXTS[name]["q"] is None else PATHS[:1]
        for env in paths:
            for k_, v in env.items():
                monkeypatch.setenv(k_, v)
            for A, B, C in cases:
                a, b, c = _coeffs(eng, A, B, C)
                outs = eng.layer_poly2(xs, a, b, c)
                assert all(o.scale == 1.0 for o in outs)
                _check_words(eng, orcs, xs, outs, A, B, C)
    finally:
        eng.close()


def test_zero_term_in_one_prime_and_absent_terms(monkeypatch):
    """A = t_0 is 0 mod the first plaintext prime only: there the output is B x + C alone; c absent, then b absent."""
    eng, orcs = _pair("n8192-cryptonets", monkeypatch)
    try:
        _, xs = _inputs(eng, 2, 2, dims=[eng.N, 100])
        t0 = CONTEXTS["n8192-cryptonets"]["t"][0]
        for A, B, C in ((t0, 5, 9), (4, -3, None), (-6, None, 17), (t0, t0, t0)):
            outs = eng.layer_poly2(xs, *_coeffs(eng, A, B, C))
            _check_words(eng, orcs, xs, outs, A, B, C)
    finally:
        eng.close()


@pytest.mark.parametrize("name", ["n4096", "n8192-cryptonets", "n16384", "n8192-int"])
def test_identity_coefficients_give_the_square(name, monkeypatch):
    eng, _ = _pair(name, monkeypatch)
    try:
        _, xs = _inputs(eng, 70, 3, bound=50)  # 70 >= 64 ciphertexts: the fused key switch by default
        monkeypatch.delenv("CNHE_KS_FUSED", raising=False)
        for fused in ("1", "0"):
            monkeypatch.setenv("CNHE_MUL_FUSED", fused)
            sq = eng.layer_square(xs)
            p2 = eng.layer_poly2(xs, *_coeffs(eng, 1, None, None))
            p0 = eng.layer_poly2(xs, *_coeffs(eng, 1, 0, 0))
            for ch in range(eng.P):
                for i in (0, 35, 69):
                    w = sq[i].export_raw(ch)
                    assert np.array_equal(p2[i].export_raw(ch), w) and np.array_equal(p0[i].export_raw(ch), w)
    finally:
        eng.close()


def test_operation_counts_are_the_composition(monkeypatch):
    eng, _ = _pair("n8192-cryptonets", monkeypatch)
    try:
        _, xs = _inputs(eng, 2, 4)
        t0 = CONTEXTS["n8192-cryptonets"]["t"][0]
        eng.op_counts(reset=True)
        eng.layer_poly2(xs, *_coeffs(eng, t0, 3, 5))  # A is 0 mod t_0: one scalar multiply fewer there
        got = eng.op_counts(reset=True)
        P, n = 2, 2
        assert got["Multiplication"] == P * n and got["Relinarization"] == P * n, got
        assert got["ScalarMultiplication"] == (P - 1) * n + P * n and got["Addition"] == P * n and got["PlainAddition"] == P * n, got
    finally:
        eng.close()


def test_two_key_slots_in_one_call():
    from cryptonets_b200.engine import DENSE, Engine
    T, N = 2277377, 8192
    server = Engine([T], N, 40, 40, 3)
    server.keygen(100)
    client = Engine([T], N, 40, 40, 3)
    client.keygen(200)
    try:
        slot = server.add_client_compact(client.save_compact_keys(public=False))
        rng = np.random.default_rng(6)
        vecs = []
        for i in range(6):
            owner = server if i % 2 == 0 else client
            v = owner.encrypt(rng.integers(0, 1000, N // 2).astype(np.float64), 1.0, DENSE)
            if owner is client:
                raw = client.export_raw_many([v])
                v.dispose()
                v = server.import_raw(np.ascontiguousarray(raw[:, 0]), 1, N // 2)
                v.set_key_slot(slot)
            vecs.append(v)
        a, b, c = _coeffs(server, 3, -2, 7)
        mixed = server.layer_poly2(vecs, a, b, c)
        alone = {s: server.layer_poly2([v for i, v in enumerate(vecs) if i % 2 == s], a, b, c) for s in (0, 1)}
        for i, o in enumerate(mixed):
            assert o.key_slot == vecs[i].key_slot
            assert np.array_equal(o.export_raw(), alone[i % 2][i // 2].export_raw())
    finally:
        client.close()
        server.close()


def test_refusals(monkeypatch):
    from cryptonets_b200.engine import DENSE, SPARSE
    eng, _ = _pair("n4096", monkeypatch)
    try:
        _, xs = _inputs(eng, 2, 5)
        a, b, c = _coeffs(eng, 2, 3, 4)

        def refused(fn):
            with pytest.raises(CnheError) as e:
                fn()
            assert e.value.code == ERR_INVALID

        refused(lambda: eng.layer_poly2([eng.plain(np.ones(4), 1.0, DENSE)], a, b, c))              # plaintext input
        refused(lambda: eng.layer_poly2(xs, eng.encrypt(np.array([2.0]), 1.0, SPARSE), b, c))     # encrypted coefficient
        refused(lambda: eng.layer_poly2(xs, eng.plain(np.array([2.0]), 1.0, DENSE), b, c))        # dense coefficient
        refused(lambda: eng.layer_poly2(xs, a, eng.plain(np.array([2.0, 1.0]), 1.0, SPARSE), c))  # dimension != 1
        refused(lambda: eng.layer_poly2(xs, a, b, eng.plain(np.array([2.0, 1.0]), 1.0, SPARSE)))
        other = eng.encrypt(np.ones(8), 2.0, DENSE)
        refused(lambda: eng.layer_poly2([xs[0], other], a, b, c))                                   # inputs of different scales
        s2 = [eng.encrypt(np.ones(8), 2.0, DENSE)]
        W = eng.plain(np.array([3.0]), 4.0, SPARSE)
        refused(lambda: eng.layer_poly2(s2, W, eng.plain(np.array([1.0]), 4.0, SPARSE), None))     # scale(b) s != W s^2
        refused(lambda: eng.layer_poly2(s2, W, None, eng.plain(np.array([1.0]), 8.0, SPARSE)))     # scale(c) != W s^2
        ok = eng.layer_poly2(s2, W, eng.plain(np.array([1.0]), 8.0, SPARSE), eng.plain(np.array([1.0]), 16.0, SPARSE))
        assert ok[0].scale == 16.0
        refused(lambda: eng.layer_poly2(xs, None, b, c))                                            # no quadratic coefficient
    finally:
        eng.close()


def _swap_square(net, coeffs, W, first=False):
    """replaces the last SquareActivation of the chain (first=True: the first) by PolyActivation(coeffs, W) and returns the new layer"""
    from cryptonets_b200.layers import PolyActivation, SquareActivation
    parents, layer = [], net
    while getattr(layer, "Source", None) is not None:
        if isinstance(layer.Source, SquareActivation):
            parents.append(layer)
        layer = layer.Source
    parent = parents[-1] if first else parents[0]
    parent.Source = PolyActivation(Source=parent.Source.Source, Coefficients=coeffs, CoefficientScale=W)
    return parent.Source


def _budget(f, m):
    vs = m.vectors if hasattr(m, "vectors") else [m]
    return min(f.engine.noise_budget(v.vec, ch, 0) for v in vs for ch in range(f.engine.P))


def _layer_chain(net):
    out, p = [], net
    while p is not None and hasattr(p, "Source"):
        out.append(p)
        p = p.Source
    return out[::-1]


def test_lola_small_with_poly_activation_equals_raw():
    """lola_small at k = 4 (the configuration that decrypts) with its square replaced: scores equal the Raw backend's exactly.  The
    first image goes layer by layer, and the noise budget entering and leaving the activation is printed next to the final one."""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import LOLA_SMALL_PRIMES, lola_small, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    coeffs, W = (0.125, 0.5, 0.25), 8.0
    f = B200BfvFactory(LOLA_SMALL_PRIMES, 8192, DecompositionBitCount=40, GaloisDecompositionBitCount=40, SmallModulusCount=4, seed=5)
    try:
        imgs = synthetic_mnist(2, seed=6)
        net, rd = lola_small(f, imgs)
        poly = _swap_square(net, coeffs, W)
        net.PrepareNetwork()
        raw_net, _ = lola_small(RawFactory(8192), imgs)
        _swap_square(raw_net, coeffs, W)
        raw_net.PrepareNetwork()
        prod_t = LOLA_SMALL_PRIMES[0] * LOLA_SMALL_PRIMES[1]
        budgets = {}
        for image in range(2):
            if image == 0:
                out = rd.GetNext()
                for layer in _layer_chain(net)[1:]:
                    out = layer.Apply(out)
                    if layer is poly.Source or layer is poly:
                        budgets["entering" if layer is poly.Source else "leaving"] = _budget(f, out)
            else:
                out = net.GetNext()
            budget = _budget(f, out)
            got = np.asarray(out.Decrypt()).reshape(-1)
            want_m = raw_net.GetNext()
            want = np.asarray(want_m.Decrypt()).reshape(-1)
            assert np.abs(np.asarray(want_m.Data)).max() < prod_t / 2
            assert budget > 0
            assert np.array_equal(got, want)
        print("lola_small PolyActivation%s W=%g: output scale %g, noise budget entering / leaving the activation %d / %d bits, final %d bits"
              % (coeffs, W, poly.GetOutputScale(), budgets["entering"], budgets["leaving"], budget))
    finally:
        f.Dispose()


def test_lola_with_poly_activation_before_duplicate_equals_raw():
    """LoLa with the square that feeds LLDuplicateLayer replaced: Duplicate rotates whole ciphertexts and adds them, so the constant term
    must leave the padding slots at zero (cnhe_layer_poly2 adds C to a vector's data slots only).  Scores agree with the Raw backend as in
    the square network's test."""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import LOLA_PRIMES, lola, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    coeffs, W = (0.5, 0.25, 0.125), 2.0
    f = B200BfvFactory(LOLA_PRIMES, 8192, seed=5)
    try:
        imgs = synthetic_mnist(2, seed=6)
        net, _ = lola(f, imgs)
        _swap_square(net, coeffs, W, first=True)
        net.PrepareNetwork()
        raw_net, _ = lola(RawFactory(8192), imgs)
        _swap_square(raw_net, coeffs, W, first=True)
        raw_net.PrepareNetwork()
        prod_t = int(np.prod([int(t) for t in LOLA_PRIMES], dtype=object))
        for _ in range(2):
            out = net.GetNext()
            budget = _budget(f, out)
            got = np.asarray(out.Decrypt()).reshape(-1)
            want_m = raw_net.GetNext()
            want = np.asarray(want_m.Decrypt()).reshape(-1)
            assert np.abs(np.asarray(want_m.Data)).max() < prod_t / 2
            assert budget > 0
            assert np.allclose(got, want, rtol=1e-9, atol=1e-9) and got.argmax() == want.argmax()
        print("lola PolyActivation%s W=%g before Duplicate: final noise budget %d bits" % (coeffs, W, budget))
    finally:
        f.Dispose()


def test_cryptonets_with_both_squares_replaced_equals_raw():
    """A small CryptoNets-MNIST batch with both squares replaced by PolyActivation: scores agree with the Raw backend (doubles: to 1e-9 of
    the largest score, as the square network's test compares) and give the same predictions."""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import CRYPTONETS_PRIMES, cryptonets_mnist, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    coeffs, W = (0.25, 0.5, 0.125), 4.0
    f = B200BfvFactory(CRYPTONETS_PRIMES, 8192, seed=77)
    try:
        imgs = synthetic_mnist(64, seed=8)
        nets = []
        for fac in (f, RawFactory(8192)):
            net, _ = cryptonets_mnist(fac, imgs, timing=False)
            for _ in range(2):
                _swap_square(net, coeffs, W)
            net.PrepareNetwork()
            nets.append(net)
        out = nets[0].GetNext()
        budget = _budget(f, out)
        scores = out.Decrypt()
        want_m = nets[1].GetNext()
        want = want_m.Decrypt()
        prod_t = CRYPTONETS_PRIMES[0] * CRYPTONETS_PRIMES[1]
        assert np.abs(np.asarray(want_m.Data)).max() < prod_t / 2
        assert budget > 0
        assert np.allclose(scores, want, rtol=1e-9, atol=1e-9 * np.abs(want).max())
        assert np.array_equal(np.argmax(scores, axis=1), np.argmax(want, axis=1))
        print("cryptonets PolyActivation%s W=%g twice: output scale %g, final noise budget %d bits" % (coeffs, W, want_m.Scale, budget))
    finally:
        f.Dispose()
