"""cnhe_layer_poly: cubic and quartic activations in two levels of squares (DESIGN.md section 4.12).

Every output word must equal the CPU oracle's composition, per plaintext prime, with the constants of test_poly4_constants.py:
  quartic  q = poly2(x; 1, beta, gamma);  y = relin(A . q^2) + D' . x + E'
  cubic    u = relin(x^2);  q1 = u + x + gamma;  y = relin(lambda . (q1^2 - u^2)) + C' . x + D'
(the size-3 difference formed here in numpy mod q_l; a term that is 0 mod the prime is skipped there), on every path the products take:
fused square or separate kernels, fused or digit key switch, the FP64 and integer floors, N = 4096 / 8192 / 16384
and 53/56-bit moduli.  (1, 0, 0, 0, 0) is the square taken twice, the cubic relinearises once per output at its second level, mixed key
slots give each client's words, and lola_small with its square replaced by a quartic or a cubic decrypts to the Raw backend."""
import numpy as np
import pytest

from cryptonets_b200._lib import CnheError
from test_poly4_constants import _is_prime, cubic_constants, quartic_constants

pytestmark = pytest.mark.gpu

ERR_INVALID = -1


def _prime(bits, N):
    c = ((1 << bits) - 1) // (2 * N) * (2 * N) + 1
    while not _is_prime(c):
        c -= 2 * N
    return c


# name: plain primes, N, decomposition bit count, coefficient moduli (None: the default), environment at context creation
CONTEXTS = {
    "n4096": dict(t=[40961], N=4096, dbc=10, q=None, env={}),
    "n8192-cryptonets": dict(t=[549764251649, 549764284417], N=8192, dbc=10, q=None, env={}),
    "n16384": dict(t=[786433], N=16384, dbc=60, q=None, env={}),
    "n8192-int": dict(t=[2277377, 2424833], N=8192, dbc=40, q=None, env={"CNHE_NTT_INT": "1"}),
    "n4096-q53": dict(t=[40961], N=4096, dbc=10, q=[_prime(53, 4096), _prime(56, 4096)], env={}),
}
PATHS = [dict(CNHE_MUL_FUSED="1", CNHE_KS_FUSED="1"), dict(CNHE_MUL_FUSED="0", CNHE_KS_FUSED="0"), dict(CNHE_MUL_FUSED="1", CNHE_KS_FUSED="0"),
         dict(CNHE_MUL_FUSED="0", CNHE_KS_FUSED="1")]


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


def _inputs(eng, seed, bound=200):
    """dense vectors with and without padding slots, and a sparse vector"""
    from cryptonets_b200.engine import DENSE, SPARSE
    rng = np.random.default_rng(seed)
    N = eng.N
    xs = [eng.encrypt(rng.integers(-bound, bound, d).astype(np.float64), 1.0, DENSE) for d in (N, N // 2 + 3, N + 5)]
    xs.append(eng.encrypt(rng.integers(-bound, bound, 3).astype(np.float64), 1.0, SPARSE))
    return xs


def _coeffs(eng, cs):
    """cs[j] the integer coefficient of x^j (None: absent) -> plain sparse vectors of dimension 1 at scale 1"""
    from cryptonets_b200.engine import SPARSE
    return [None if v is None else eng.plain(np.array([float(v)]), 1.0, SPARSE) for v in cs]


def _sub3(orc, a, b):
    q = np.array(orc.q, dtype=np.uint64).reshape(1, -1, 1)
    a, b = a.reshape(3, orc.k, orc.N), b.reshape(3, orc.k, orc.N)
    return ((a + (q - b)) % q).astype(np.uint64).ravel()


def _const(orc, v, fill):
    """add_plain's plaintext for the constant v: the constant polynomial, or v in the first `fill` slots only"""
    return [v] if fill is None else orc.encode(np.where(np.arange(orc.N) < fill, v, 0).astype(np.uint64))


def _oracle_words(orc, x, cs, fill):
    t = orc.t
    r = [0 if v is None else v % t for v in cs]
    out = None
    if len(cs) == 5:
        beta, gamma, D1, E1 = quartic_constants(t, *r[::-1])
        q = orc.relinearize(orc.multiply_plain(orc.multiply(x, x), [1]))
        if beta:
            q = orc.add(q, orc.multiply_plain(x, [beta]))
        if gamma:
            q = orc.add_plain(q, _const(orc, gamma, fill))
        out = orc.relinearize(orc.multiply_plain(orc.multiply(q, q), [r[4]]))
        lin, cst = D1, E1
    else:
        lam, gamma, C1, D1 = cubic_constants(t, *r[::-1])
        u = orc.relinearize(orc.multiply(x, x))
        q1 = orc.add(u, x)
        if gamma:
            q1 = orc.add_plain(q1, _const(orc, gamma, fill))
        out = orc.relinearize(orc.multiply_plain(_sub3(orc, orc.multiply(q1, q1), orc.multiply(u, u)), [lam]))
        lin, cst = C1, D1
    if lin:
        out = orc.add(out, orc.multiply_plain(x, [lin]))
    if cst:
        out = orc.add_plain(out, _const(orc, cst, fill))
    return out


def _check_words(eng, orcs, xs, outs, cs):
    from cryptonets_b200.engine import DENSE
    for ch, orc in enumerate(orcs):
        for x, o in zip(xs, outs):
            assert o.blocks == x.blocks and o.dim == x.dim
            for bl in range(x.blocks):
                dense_fill = x.format == DENSE and bl == x.blocks - 1 and x.dim % eng.N
                fill = x.dim % eng.N if dense_fill else None
                assert np.array_equal(o.export_raw(ch, bl), _oracle_words(orc, x.export_raw(ch, bl), cs, fill)), (ch, bl, cs)


@pytest.mark.parametrize("name", list(CONTEXTS))
def test_words_equal_oracle_composition(name, monkeypatch):
    eng, orcs = _pair(name, monkeypatch)
    try:
        xs = _inputs(eng, 1)
        t0 = CONTEXTS[name]["t"][0]
        # coefficients of x^0 .. x^d: negative values, constants in the upper half of t, absent middle terms
        cases = [[t0 // 2 + 5, -7, 3, -2, 5], [-11, None, None, None, 3], [t0 // 2 + 9, 4, -6, 2], [None, 5, None, -3]]
        paths = PATHS if eng.N <= 8192 and not CONTEXTS[name]["env"] and CONTEXTS[name]["q"] is None else PATHS[:1]
        for env in paths:
            for k_, v in env.items():
                monkeypatch.setenv(k_, v)
            for cs in cases:
                outs = eng.layer_poly(xs, _coeffs(eng, cs))
                assert all(o.scale == 1.0 for o in outs)
                _check_words(eng, orcs, xs, outs, cs)
    finally:
        eng.close()


@pytest.mark.parametrize("name", ["n4096", "n8192-cryptonets", "n16384", "n8192-int"])
def test_identity_quartic_is_the_square_twice(name, monkeypatch):
    eng, _ = _pair(name, monkeypatch)
    try:
        from cryptonets_b200.engine import DENSE
        rng = np.random.default_rng(3)
        xs = [eng.encrypt(rng.integers(-20, 20, eng.N).astype(np.float64), 1.0, DENSE) for _ in range(70)]  # the fused key switch
        monkeypatch.delenv("CNHE_KS_FUSED", raising=False)
        for fused in ("1", "0"):
            monkeypatch.setenv("CNHE_MUL_FUSED", fused)
            sq = eng.layer_square(eng.layer_square(xs))
            p4 = eng.layer_poly(xs, _coeffs(eng, [None, None, None, None, 1]))
            p0 = eng.layer_poly(xs, _coeffs(eng, [0, 0, 0, 0, 1]))
            for ch in range(eng.P):
                for i in (0, 35, 69):
                    w = sq[i].export_raw(ch)
                    assert np.array_equal(p4[i].export_raw(ch), w) and np.array_equal(p0[i].export_raw(ch), w)
    finally:
        eng.close()


def test_operation_counts_are_the_composition(monkeypatch):
    eng, _ = _pair("n8192-cryptonets", monkeypatch)
    try:
        from cryptonets_b200.engine import DENSE
        xs = [eng.encrypt(np.arange(8.0), 1.0, DENSE) for _ in range(3)]
        P, n = 2, 3
        eng.op_counts(reset=True)
        eng.layer_poly(xs, _coeffs(eng, [5, 4, 3, 2, 1]))
        got = eng.op_counts(reset=True)
        # every term nonzero in both channels (checked against the constants): level 1 = poly2(1, beta, gamma), level 2 = A, D', E'
        for t in CONTEXTS["n8192-cryptonets"]["t"]:
            assert all(quartic_constants(t, 1, 2, 3, 4, 5))
        assert got["Multiplication"] == 2 * P * n and got["Relinarization"] == 2 * P * n, got
        assert got["ScalarMultiplication"] == 4 * P * n and got["Addition"] == 2 * P * n and got["PlainAddition"] == 2 * P * n, got
        eng.layer_poly(xs, _coeffs(eng, [5, 4, 3, 2]))
        got = eng.op_counts(reset=True)
        for t in CONTEXTS["n8192-cryptonets"]["t"]:
            assert all(cubic_constants(t, 2, 3, 4, 5))
        # level 1: square + relin, add, add_plain; level 2: two squares, subtract, lambda, one relin, C' x (scalar + add), D'
        assert got["Multiplication"] == 3 * P * n and got["Relinarization"] == 2 * P * n, got
        assert got["Subtraction"] == P * n and got["ScalarMultiplication"] == 2 * P * n, got
        assert got["Addition"] == 2 * P * n and got["PlainAddition"] == 2 * P * n, got
    finally:
        eng.close()


def test_cubic_second_level_relinearises_once_per_output(monkeypatch):
    """the pair floor: q1^2 and u^2 are combined before the key switch, so the cubic launches the key switch as often as two squares"""
    eng, _ = _pair("n8192-cryptonets", monkeypatch)
    try:
        from cryptonets_b200.engine import DENSE
        rng = np.random.default_rng(4)
        xs = [eng.encrypt(rng.integers(-50, 50, eng.N).astype(np.float64), 1.0, DENSE) for _ in range(8)]
        cs = _coeffs(eng, [1, 2, 3, 4])
        eng.layer_poly(xs, cs)  # warm
        for ks in ("1", "0"):
            monkeypatch.setenv("CNHE_KS_FUSED", ks)
            launches = {}
            for what, fn in (("cubic", lambda: eng.layer_poly(xs, cs)), ("two squares", lambda: eng.layer_square(eng.layer_square(xs)))):
                eng.prof_enable(True)
                eng.op_counts(reset=True)
                fn()
                got = eng.op_counts(reset=True)
                prof = eng.prof_collect()
                eng.prof_enable(False)
                assert got["Relinarization"] == 2 * eng.P * len(xs), (what, got)
                launches[what] = prof["keyswitch_mac"]["launches"]
            assert launches["cubic"] == launches["two squares"] > 0, launches
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
            v = owner.encrypt(rng.integers(0, 100, N // 2).astype(np.float64), 1.0, DENSE)
            if owner is client:
                raw = client.export_raw_many([v])
                v.dispose()
                v = server.import_raw(np.ascontiguousarray(raw[:, 0]), 1, N // 2)
                v.set_key_slot(slot)
            vecs.append(v)
        for cs in ([7, -2, 3, 1, 2], [7, -2, 3, 4]):
            co = _coeffs(server, cs)
            mixed = server.layer_poly(vecs, co)
            alone = {s: server.layer_poly([v for i, v in enumerate(vecs) if i % 2 == s], co) for s in (0, 1)}
            for i, o in enumerate(mixed):
                assert o.key_slot == vecs[i].key_slot
                assert np.array_equal(o.export_raw(), alone[i % 2][i // 2].export_raw())
    finally:
        client.close()
        server.close()


def test_refusals_leave_the_context_usable(monkeypatch):
    from cryptonets_b200.engine import DENSE, SPARSE
    eng, orcs = _pair("n8192-cryptonets", monkeypatch)
    try:
        xs = _inputs(eng, 5)[:2]
        cs = _coeffs(eng, [4, 3, 2, 1, 2])
        t0, t1 = CONTEXTS["n8192-cryptonets"]["t"]

        def refused(fn, text=None):
            with pytest.raises(CnheError) as e:
                fn()
            assert e.value.code == ERR_INVALID
            if text:
                assert text in str(e.value), str(e.value)

        refused(lambda: eng.layer_poly(xs, cs[:3]))                                                   # degree 2
        refused(lambda: eng.layer_poly(xs, cs + cs[:1]))                                              # degree 5
        refused(lambda: eng.layer_poly(xs, cs[:4] + [None]))                                          # no leading coefficient
        refused(lambda: eng.layer_poly(xs, cs[:4] + _coeffs(eng, [t1])), str(t1))                     # 0 mod the second prime
        refused(lambda: eng.layer_poly(xs, cs[:3] + _coeffs(eng, [2 * t0])), str(t0))                 # cubic, 0 mod the first
        refused(lambda: eng.layer_poly(xs, cs[:4] + [eng.encrypt(np.array([2.0]), 1.0, SPARSE)]))     # encrypted coefficient
        refused(lambda: eng.layer_poly(xs, [eng.plain(np.array([2.0]), 1.0, DENSE)] + cs[1:]))        # dense coefficient
        refused(lambda: eng.layer_poly(xs, [eng.plain(np.array([2.0, 1.0]), 1.0, SPARSE)] + cs[1:]))  # dimension != 1
        refused(lambda: eng.layer_poly([eng.plain(np.ones(4), 1.0, DENSE)], cs))                      # plaintext input
        refused(lambda: eng.layer_poly([xs[0], eng.encrypt(np.ones(8), 2.0, DENSE)], cs))             # inputs of different scales
        s2 = [eng.encrypt(np.ones(8), 2.0, DENSE)]
        W = 3.0
        good = [eng.plain(np.array([1.0]), W * 2.0 ** (4 - j), SPARSE) for j in range(5)]
        for j in range(4):
            bad = list(good)
            bad[j] = eng.plain(np.array([1.0]), W * 2.0 ** (3 - j), SPARSE)
            refused(lambda: eng.layer_poly(s2, bad))                                                  # scale(c_j) != W s^(4 - j)
        assert eng.layer_poly(s2, good)[0].scale == W * 16.0
        assert eng.layer_poly(s2, [eng.plain(np.array([1.0]), W * 2.0 ** (3 - j), SPARSE) for j in range(4)])[0].scale == W * 8.0
        # the context still computes the right words
        outs = eng.layer_poly(xs, cs)
        _check_words(eng, orcs, xs, outs, [4, 3, 2, 1, 2])
    finally:
        eng.close()


def _swap_square(net, coeffs, W):
    """replaces the last SquareActivation of the chain by PolyActivation(coeffs, W) and returns the new layer"""
    from cryptonets_b200.layers import PolyActivation, SquareActivation
    layer = net
    while getattr(layer, "Source", None) is not None:
        if isinstance(layer.Source, SquareActivation):
            layer.Source = PolyActivation(Source=layer.Source.Source, Coefficients=coeffs, CoefficientScale=W)
            return layer.Source
        layer = layer.Source
    raise AssertionError("no square")


def _budget(f, m):
    vs = m.vectors if hasattr(m, "vectors") else [m]
    return min(f.engine.noise_budget(v.vec, ch, 0) for v in vs for ch in range(f.engine.P))


def _layer_chain(net):
    out, p = [], net
    while p is not None and hasattr(p, "Source"):
        out.append(p)
        p = p.Source
    return out[::-1]


def _primes_1_mod(m, bits, count):
    out, c = [], (1 << bits) // m * m + 1
    while len(out) < count:
        if _is_prime(c):
            out.append(c)
        c += m
    return out


# a quartic fit of ReLU on [-1, 1] (least squares on the Chebyshev nodes) and an odd cubic (a sigmoid-style output), highest degree first
QUARTIC_RELU = (-0.4453, 0.0, 0.9375, 0.5, 0.0469)
CUBIC = (-0.0625, 0.0, 0.5, 0.25)


@pytest.mark.parametrize("coeffs, W", [(QUARTIC_RELU, 16.0), (CUBIC, 16.0)])
def test_lola_small_with_cubic_or_quartic_equals_raw(coeffs, W):
    """lola_small (N = 8192, k = 5) with its square replaced: enough ~20-bit plaintext primes that the Raw backend's largest |value| is
    below half their product; the scores equal the Raw backend's.  The noise budgets entering and leaving the activation and at the
    scores are printed."""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import lola_small, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    imgs = synthetic_mnist(2, seed=6)
    raw_net, _ = lola_small(RawFactory(8192), imgs)
    _swap_square(raw_net, coeffs, W)
    raw_net.PrepareNetwork()
    peak, want = 0.0, []
    for _ in range(2):
        m = raw_net.GetNext()  # the chain's largest value is at the activation or after it; the scores are checked below
        peak = max(peak, float(np.abs(np.asarray(m.Data)).max()))
        want.append(m)
    raw_first, _ = lola_small(RawFactory(8192), imgs)
    _swap_square(raw_first, coeffs, W)
    raw_first.PrepareNetwork()
    out = None
    for layer in _layer_chain(raw_first):  # every intermediate of the first image
        out = layer.GetNext() if out is None else layer.Apply(out)
        peak = max(peak, float(np.abs(np.asarray(out.Data)).max()))
    primes, prod = [], 1
    for p in _primes_1_mod(2 * 8192, 20, 12):
        if prod >= 4 * peak:
            break
        primes.append(p)
        prod *= p
    assert peak < prod / 2, (peak, prod)
    f = B200BfvFactory(primes, 8192, DecompositionBitCount=40, GaloisDecompositionBitCount=40, SmallModulusCount=5, seed=5)
    try:
        net, rd = lola_small(f, imgs)
        poly = _swap_square(net, coeffs, W)
        net.PrepareNetwork()
        budgets = {}
        for image in range(2):
            if image == 0:
                o = rd.GetNext()
                for layer in _layer_chain(net)[1:]:
                    o = layer.Apply(o)
                    if layer is poly.Source or layer is poly:
                        budgets["entering" if layer is poly.Source else "leaving"] = _budget(f, o)
            else:
                o = net.GetNext()
            budget = _budget(f, o)
            got = np.asarray(o.Decrypt()).reshape(-1)
            w = np.asarray(want[image].Decrypt()).reshape(-1)
            assert budget > 0
            assert np.allclose(got, w, rtol=1e-9, atol=1e-9 * np.abs(w).max()) and got.argmax() == w.argmax()
        print("lola_small PolyActivation%s W=%g: %d plaintext primes of ~20 bits (largest |value| %.3g < prod/2 = %.3g), output scale %g, "
              "noise budget entering / leaving the activation %d / %d bits, at the scores %d bits"
              % (coeffs, W, len(primes), peak, prod / 2, poly.GetOutputScale(), budgets["entering"], budgets["leaving"], budget))
    finally:
        f.Dispose()
