"""cnhe_layer_activation_conv_dense: the square or quadratic activation, the scalar MAC on the size-3 products, then one relinearisation
per output.

Every output word must equal the CPU oracle's composition, per plaintext prime:
    P3 = A . multiply(x, x) + (B x0 + C, B x1, 0),   out[m] = relinearize(mac(c0, c1) + bias, mac(c2))
on every product path (fused square or separate kernels), both key-switch paths, N = 4096 / 8192 / 16384, every scalar-MAC kernel
(wgmma, mma.sync, FP64, 128-bit integer) and moduli of 53/56 bits.  Operation counts are the composition's, two key slots equal per-slot
calls, every refusal creates no vector, and CryptoNets-MNIST with deferred relinearisation decrypts to the default network's scores."""
import ctypes as C
import os

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


CONTEXTS = {
    "n4096": dict(t=[40961], N=4096, dbc=10, q=None),
    "n8192-cryptonets": dict(t=[549764251649, 549764284417], N=8192, dbc=10, q=None),
    "n16384": dict(t=[786433], N=16384, dbc=60, q=None),
    "n4096-q53": dict(t=[40961], N=4096, dbc=10, q=[_prime(53, 4096), _prime(56, 4096)]),
}
PATHS = [dict(CNHE_MUL_FUSED="1", CNHE_KS_FUSED="1"), dict(CNHE_MUL_FUSED="0", CNHE_KS_FUSED="0"), dict(CNHE_MUL_FUSED="1", CNHE_KS_FUSED="0"),
         dict(CNHE_MUL_FUSED="0", CNHE_KS_FUSED="1")]
KERNEL_ENV = ("CNHE_MAC_NO_UMMA", "CNHE_MAC_NO_IMMA", "CNHE_MAC_INT", "CNHE_MUL_FUSED", "CNHE_KS_FUSED")


def _pair(name, monkeypatch):
    from cryptonets_b200.engine import Engine
    from oracle.oracle_py import Oracle
    cfg = CONTEXTS[name]
    for var in KERNEL_ENV:
        monkeypatch.delenv(var, raising=False)
    eng = Engine(cfg["t"], cfg["N"], cfg["dbc"], 20, -1, coeff_moduli=cfg["q"])
    eng.keygen(31)
    orcs = []
    for ch, t in enumerate(cfg["t"]):
        o = Oracle(t, cfg["N"], -1, cfg["dbc"], 20, custom_q=cfg["q"])
        o.keygen(31 + ch)
        orcs.append(o)
    return eng, orcs


def _inputs(eng, n, dim, seed, bound=100):
    from cryptonets_b200.engine import DENSE
    rng = np.random.default_rng(seed)
    return [eng.encrypt(rng.integers(-bound, bound, dim).astype(np.float64), 1.0, DENSE) for _ in range(n)]


def _coeffs(eng, A, B, C):
    from cryptonets_b200.engine import SPARSE
    mk = lambda v: None if v is None else eng.plain(np.array([float(v)]), 1.0, SPARSE)
    return mk(A), mk(B), mk(C)


def _lift(v, t):
    v = np.asarray(v, dtype=object) % t
    return np.array([int(x) for x in np.ravel(v)], dtype=np.uint64).reshape(np.shape(v))


class Layer:
    """one call's layer: gather [M][K], integer weights [M][K], bias per output (a constant, or an array of dim values), and the squares
    of the inputs on the oracle (cached: they do not depend on the activation's coefficients or the paths)"""

    def __init__(self, eng, orcs, xs, gather, w, bias):
        from cryptonets_b200.engine import DENSE, SPARSE
        self.eng, self.orcs, self.xs, self.gather, self.w, self.bias = eng, orcs, xs, np.asarray(gather, np.int32), np.asarray(w), bias
        self.M, self.K = self.w.shape
        self.wv = [eng.plain(self.w[m].astype(np.float64), 1.0, SPARSE) for m in range(self.M)]
        dim = xs[0].dim
        self.bias_vals = None if bias is None else [np.full(dim, float(b)) if np.isscalar(b) else np.asarray(b, np.float64) for b in bias]
        self.bv = None if bias is None else [eng.plain(v, 1.0, DENSE) for v in self.bias_vals]
        self._sq, self._want = {}, {}

    def square(self, ch, i, bl):
        key = (ch, i, bl)
        if key not in self._sq:
            x = self.xs[i].export_raw(ch, bl)
            self._sq[key] = (x, self.orcs[ch].multiply(x, x))
        return self._sq[key]

    def run(self, coeffs):
        a, b, c = coeffs if coeffs is not None else (None, None, None)
        return self.eng.layer_activation_conv_dense(self.xs, a, b, c, self.gather, self.wv, self.bv, self.M, self.K)

    def want(self, ch, bl, A, B, C, outputs):
        """oracle words of the given outputs, block bl, channel ch; A, B, C integers or None (A = "square": the square); the same for
        every path, so computed once"""
        key = (ch, bl, A, B, C, tuple(outputs))
        if key not in self._want:
            self._want[key] = self._compose(ch, bl, A, B, C, outputs)
        return self._want[key]

    def _compose(self, ch, bl, A, B, C, outputs):
        orc, N = self.orcs[ch], self.eng.N
        t, k = orc.t, orc.k
        kN = k * N
        dim = self.xs[0].dim
        fill = dim % N if bl == self.xs[0].blocks - 1 and dim % N else None
        p3s = []
        for i in range(len(self.xs)):
            x, sq = self.square(ch, i, bl)
            if A == "square":
                p3s.append(sq)
                continue
            Am, Bm, Cm = (None if v is None or v % t == 0 else v % t for v in (A, B, C))
            p3 = orc.multiply_plain(sq, [Am]) if Am is not None else np.zeros(3 * kN, np.uint64)
            lo = p3[:2 * kN].copy()
            if Bm is not None:
                lo = orc.add(lo, orc.multiply_plain(x, [Bm]))
            if Cm is not None:
                lo = orc.add_plain(lo, [Cm] if fill is None else orc.encode(np.where(np.arange(N) < fill, Cm, 0).astype(np.uint64)))
            p3s.append(np.concatenate([lo, p3[2 * kN:]]))
        p3s = np.stack(p3s)
        wres = _lift(self.w, t)
        # a dense plaintext is the constant polynomial only when it fills every slot; otherwise its padding slots stay zero
        const = self.bias is not None and all(np.isscalar(b) for b in self.bias) and dim % N == 0
        bres = _lift(np.array(self.bias, dtype=object), t) if const else None
        c01 = orc.mac_layer(p3s[:, :2 * kN], self.gather, wres, bres, self.M, self.K, threads=max(4, os.cpu_count() or 1)).reshape(self.M, -1)
        c2in = np.concatenate([p3s[:, 2 * kN:], np.zeros((len(self.xs), kN), np.uint64)], axis=1)
        c2 = orc.mac_layer(c2in, self.gather, wres, None, self.M, self.K, threads=max(4, os.cpu_count() or 1)).reshape(self.M, -1)[:, :kN]
        out = {}
        for m in outputs:
            lo = c01[m]
            if self.bias is not None and not const:
                vals = np.zeros(N)
                part = self.bias_vals[m][bl * N:(bl + 1) * N]
                vals[:len(part)] = part
                lo = orc.add_plain(lo, orc.encode(_lift(vals, t)))
            out[m] = orc.relinearize(np.concatenate([lo, c2[m]]))
        return out

    def check(self, outs, A, B, C, outputs=None):
        outputs = range(self.M) if outputs is None else outputs
        for ch in range(self.eng.P):
            for bl in range(self.xs[0].blocks):
                want = self.want(ch, bl, A, B, C, outputs)
                for m in outputs:
                    assert np.array_equal(outs[m].export_raw(ch, bl), want[m]), (ch, bl, m)


def _conv_gather(rng, n_in, M, K, padded=True):
    g = rng.integers(-1 if padded else 0, n_in, (M, K)).astype(np.int32)
    g[:, 0] = np.arange(M) % n_in
    return g


def _weights(rng, M, K, bound=120):
    w = rng.integers(-bound, bound + 1, (M, K))
    w[:, 0] = np.where(w[:, 0] == 0, 7, w[:, 0])
    return w


@pytest.mark.parametrize("name", ["n4096", "n8192-cryptonets", "n16384"])
def test_words_equal_oracle_composition(name, monkeypatch):
    """M = 10 (convolution-shaped gather with padded taps) and M = 66 (dense, >= 64 outputs: the fused key switch by default) on every
    product and key-switch path; the square, a quadratic with C in the upper half of t, one with b absent and one whose A is 0 mod one
    prime.  The inputs' last slots are padding, so C goes to the data slots only."""
    eng, orcs = _pair(name, monkeypatch)
    try:
        N, ts = eng.N, CONTEXTS[name]["t"]
        rng = np.random.default_rng(5)
        n_in = 12
        xs = _inputs(eng, n_in, N - 5, 1)
        conv = Layer(eng, orcs, xs, _conv_gather(rng, n_in, 10, 6), _weights(rng, 10, 6), list(rng.integers(-500, 500, 10)))
        dense = Layer(eng, orcs, xs, np.tile(np.arange(n_in, dtype=np.int32), (66, 1)), _weights(rng, 66, n_in), list(rng.integers(-500, 500, 66)))
        cases = [("square", None, None), (3, -7, ts[0] // 2 + 5), (-2, None, -11)]
        if len(ts) > 1:
            cases.append((ts[0], 5, 9))  # A = 0 mod the first prime: there P3 is B x + C alone
        paths = PATHS if N <= 8192 else PATHS[:1]
        for env in paths:
            for k_, v in env.items():
                monkeypatch.setenv(k_, v)
            for A, B, C in cases:
                coeffs = None if A == "square" else _coeffs(eng, A, B, C)
                conv.check(conv.run(coeffs), A, B, C)
                outs = dense.run(coeffs)
                assert all(o.scale == 1.0 for o in outs)
                dense.check(outs, A, B, C, outputs=[0, 1, 33, 65])
    finally:
        eng.close()


@pytest.mark.parametrize("variant", ["wgmma", "mma-sync", "fp64-env", "fp64-wide", "int", "two-blocks", "q53"])
def test_every_mac_kernel(variant, monkeypatch, capfd):
    """Each scalar-MAC kernel on the size-3 products: wgmma (slab inputs, |w| <= 254, M >= 8), mma.sync (CNHE_MAC_NO_UMMA), FP64 (|w| > 254
    or CNHE_MAC_NO_IMMA), the 128-bit integer MAC (CNHE_MAC_INT, and moduli of 53/56 bits); two-block inputs with padded taps.  Constant
    and non-constant biases alternate."""
    eng, orcs = _pair("n4096-q53" if variant == "q53" else "n4096", monkeypatch)
    try:
        N = eng.N
        rng = np.random.default_rng(sum(map(ord, variant)))
        n_in, M = 40, 16
        dim = N + 7 if variant == "two-blocks" else N
        xs = _inputs(eng, n_in, dim, 2)
        row = np.arange(n_in, dtype=np.int32)
        if variant == "two-blocks":
            row[5] = -1
        w = _weights(rng, M, n_in, 300 if variant == "fp64-wide" else 120)
        if variant != "fp64-wide":
            w[:, 1], w[:, 2] = 254, -254
        const_bias = variant in ("wgmma", "fp64-env", "int")
        bias = list(rng.integers(-900, 900, M)) if const_bias else [rng.integers(-900, 900, dim) for _ in range(M)]
        layer = Layer(eng, orcs, xs, np.tile(row, (M, 1)), w, bias)
        env = {"mma-sync": "CNHE_MAC_NO_UMMA", "fp64-env": "CNHE_MAC_NO_IMMA", "int": "CNHE_MAC_INT"}.get(variant)
        if env:
            monkeypatch.setenv(env, "1")
        monkeypatch.setenv("CNHE_UMMA_PROF", "1")  # the wgmma launcher reports itself on stderr
        capfd.readouterr()
        for A, B, C in (("square", None, None), (2, -3, 5)):
            outs = layer.run(None if A == "square" else _coeffs(eng, A, B, C))
            eng.sync()
            served = "[umma " in capfd.readouterr().err
            assert served == (variant == "wgmma"), "wrong kernel served the layer"
            layer.check(outs, A, B, C)
    finally:
        eng.close()


def test_operation_counts_are_the_composition(monkeypatch):
    """Counts equal poly2 (or square) + conv_dense, with one relinearisation per output block instead of one per input block."""
    eng, _ = _pair("n8192-cryptonets", monkeypatch)
    try:
        from cryptonets_b200.engine import DENSE, SPARSE
        rng = np.random.default_rng(7)
        n_in, M, K, P = 9, 5, 4, eng.P
        xs = _inputs(eng, n_in, eng.N + 3, 3)  # two blocks
        gather = _conv_gather(rng, n_in, M, K)
        wv = [eng.plain(w.astype(np.float64), 1.0, SPARSE) for w in _weights(rng, M, K)]
        bv = [eng.plain(np.full(eng.N + 3, 3.0), 1.0, DENSE) for _ in range(M)]
        t0 = CONTEXTS["n8192-cryptonets"]["t"][0]
        for coeffs in (None, _coeffs(eng, t0, 3, 5)):  # A is 0 mod t_0: one scalar multiply fewer there
            eng.op_counts(reset=True)
            mid = eng.layer_square(xs) if coeffs is None else eng.layer_poly2(xs, *coeffs)
            eng.layer_conv_dense(mid, gather, wv, bv, M, K)
            want = eng.op_counts(reset=True)
            want["Relinarization"] = P * M * 2
            eng.layer_activation_conv_dense(xs, *(coeffs or (None, None, None)), gather, wv, bv, M, K)
            got = eng.op_counts(reset=True)
            assert got["Multiplication"] == P * n_in * 2 and got == want, (got, want)
    finally:
        eng.close()


def test_two_key_slots_in_one_call():
    """Inputs of two clients side by side, each output's taps inside one client's columns: the outputs equal per-slot calls word for word
    and take their taps' slot; an output whose taps span both slots is refused."""
    from cryptonets_b200.engine import DENSE, SPARSE, Engine
    T, N = 2277377, 8192
    server = Engine([T], N, 40, 40, 3)
    server.keygen(100)
    client = Engine([T], N, 40, 40, 3)
    client.keygen(200)
    try:
        slot = server.add_client_compact(client.save_compact_keys(public=False))
        rng = np.random.default_rng(6)
        vecs = []
        for i in range(8):
            owner = server if i % 2 == 0 else client
            v = owner.encrypt(rng.integers(-300, 300, N // 2).astype(np.float64), 1.0, DENSE)
            if owner is client:
                raw = client.export_raw_many([v])
                v.dispose()
                v = server.import_raw(np.ascontiguousarray(raw[:, 0]), 1, N // 2)
                v.set_key_slot(slot)
            vecs.append(v)
        M, K = 6, 3
        local = rng.integers(0, 4, (M, K))                          # tap j of output m: input 2 * local + (m % 2) of slot m % 2
        gather = (2 * local + (np.arange(M) % 2)[:, None]).astype(np.int32)
        w = _weights(rng, M, K)
        wv = [server.plain(w[m].astype(np.float64), 1.0, SPARSE) for m in range(M)]
        bv = [server.plain(np.full(N // 2, float(m)), 1.0, DENSE) for m in range(M)]
        a, b, c = _coeffs(server, 3, -2, 7)
        mixed = server.layer_activation_conv_dense(vecs, a, b, c, gather, wv, bv, M, K)
        for s in (0, 1):
            ms = [m for m in range(M) if m % 2 == s]
            alone = server.layer_activation_conv_dense(vecs[s::2], a, b, c, local[ms].astype(np.int32), [wv[m] for m in ms], [bv[m] for m in ms],
                                                       len(ms), K)
            for j, m in enumerate(ms):
                assert mixed[m].key_slot == vecs[s].key_slot
                assert np.array_equal(mixed[m].export_raw(), alone[j].export_raw()), m
        bad = gather.copy()
        bad[0, 1] = 1
        with pytest.raises(CnheError) as e:
            server.layer_activation_conv_dense(vecs, a, b, c, bad, wv, bv, M, K)
        assert e.value.code == ERR_INVALID
    finally:
        client.close()
        server.close()


def _raw_call(eng, ins, a, b, c, gather, weights, bias, M, K):
    """the C call itself, so that a refusal can be seen to leave every output slot NULL"""
    from cryptonets_b200._lib import VECP
    arr = lambda vs: None if vs is None else (VECP * len(vs))(*[v.h for v in vs])
    h = lambda v: None if v is None else v.h
    g = None if gather is None else np.ascontiguousarray(gather, dtype=np.int32)
    out = (VECP * M)()
    rc = eng.L.cnhe_layer_activation_conv_dense(eng.h, arr(ins), len(ins), h(a), h(b), h(c),
                                                None if g is None else g.ctypes.data_as(C.POINTER(C.c_int32)), arr(weights), arr(bias), M, K, out)
    return rc, [out[i] for i in range(M)]


def test_refusals(monkeypatch):
    from cryptonets_b200.engine import DENSE, SPARSE
    eng, _ = _pair("n8192-cryptonets", monkeypatch)
    try:
        N, t0 = eng.N, CONTEXTS["n8192-cryptonets"]["t"][0]
        xs = _inputs(eng, 4, N, 4)
        gather = np.array([[0, 1], [2, 3]], np.int32)
        wv = [eng.plain(np.array([2.0, -3.0]), 1.0, SPARSE) for _ in range(2)]
        bv = [eng.plain(np.full(N, 1.0), 1.0, DENSE) for _ in range(2)]
        a, b, c = _coeffs(eng, 2, 3, 4)
        W = eng.plain(np.array([3.0]), 4.0, SPARSE)
        huge = 2 ** 30 // (3 * eng.k * N) + 1  # size-3 products beyond 8 GiB (the same input, listed over and over)
        cases = {
            "plaintext input": ([eng.plain(np.ones(N), 1.0, DENSE)] * 4, a, b, c, gather, wv, bv, 2, 2),
            "sparse input": ([eng.encrypt(np.ones(4), 1.0, SPARSE)] * 4, a, b, c, gather, wv, bv, 2, 2),
            "encrypted coefficient": (xs, eng.encrypt(np.array([2.0]), 1.0, SPARSE), b, c, gather, wv, bv, 2, 2),
            "dense coefficient": (xs, eng.plain(np.array([2.0]), 1.0, DENSE), b, c, gather, wv, bv, 2, 2),
            "coefficient of dimension 2": (xs, a, eng.plain(np.array([2.0, 1.0]), 1.0, SPARSE), c, gather, wv, bv, 2, 2),
            "b without a": (xs, None, b, None, gather, wv, bv, 2, 2),
            "scale(b) s != W s^2": (xs, W, eng.plain(np.array([1.0]), 1.0, SPARSE), None, gather, wv, bv, 2, 2),
            "bias scale != W s^2 scale(w)": (xs, W, None, None, gather, wv, bv, 2, 2),
            "inputs of two scales": (xs[:3] + [eng.encrypt(np.ones(N), 2.0, DENSE)], a, b, c, gather, wv, bv, 2, 2),
            "gather out of range": (xs, a, b, c, np.array([[0, 1], [2, 4]], np.int32), wv, bv, 2, 2),
            "weights of the wrong dimension": (xs, a, b, c, gather, [eng.plain(np.array([1.0, 2.0, 3.0]), 1.0, SPARSE)] * 2, bv, 2, 2),
            "empty sum mod one prime": (xs, a, b, c, gather, [wv[0], eng.plain(np.array([float(t0), 0.0]), 1.0, SPARSE)], bv, 2, 2),
            "all taps padded": (xs, a, b, c, np.array([[0, 1], [-1, -1]], np.int32), wv, bv, 2, 2),
            "bias of another dimension": (xs, a, b, c, gather, wv, [eng.plain(np.full(N // 2, 1.0), 1.0, DENSE)] * 2, 2, 2),
            "empty layer": ([], a, b, c, gather, wv, bv, 2, 2),
            "size-3 products beyond 8 GiB": ([xs[0]] * huge, None, None, None, None, [eng.plain(np.ones(1), 1.0, SPARSE)], None, 1, 1),
        }
        for what, args in cases.items():
            rc, outs = _raw_call(eng, *args)
            assert rc == ERR_INVALID, what
            assert all(o is None for o in outs), what
        ok = eng.layer_activation_conv_dense(xs, W, None, None, gather, wv, [eng.plain(np.full(N, 1.0), 4.0, DENSE)] * 2, 2, 2)
        assert ok[0].scale == 4.0
    finally:
        eng.close()


def _budget(f, m):
    vs = m.vectors if hasattr(m, "vectors") else [m]
    return min(f.engine.noise_budget(v.vec, ch, 0) for v in vs for ch in range(f.engine.P))


def _swap_squares(net, coeffs, W):
    from cryptonets_b200.layers import PolyActivation, SquareActivation
    layer = net
    while getattr(layer, "Source", None) is not None:
        if isinstance(layer.Source, SquareActivation):
            layer.Source = PolyActivation(Source=layer.Source.Source, Coefficients=coeffs, CoefficientScale=W)
        layer = layer.Source


@pytest.mark.parametrize("activation", ["square", "poly"])
def test_cryptonets_deferred_equals_default_and_raw(activation, capsys):
    """CryptoNets-MNIST at the reference parameters: the deferred network decrypts to the default network's scores exactly and to the Raw
    backend's (doubles: to 1e-9 of the largest score, with the same predictions), with both squares or both replaced by PolyActivation.
    The deferred scores' noise budget is at most 1 bit below the default's."""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import CRYPTONETS_PRIMES, cryptonets_mnist, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    coeffs, W = (0.25, 0.5, 0.125), 4.0
    f = B200BfvFactory(CRYPTONETS_PRIMES, 8192, seed=77)
    try:
        imgs = synthetic_mnist(256, seed=9)
        res = {}
        for arm, fac, defer in (("default", f, False), ("deferred", f, True), ("raw", RawFactory(8192), True)):
            net, _ = cryptonets_mnist(fac, imgs, timing=False, defer_relinearization=defer)
            if activation == "poly":
                _swap_squares(net, coeffs, W)
            net.PrepareNetwork()
            if fac is f:
                f.engine.op_counts(reset=True)
            out = net.GetNext()
            res[arm] = (np.asarray(out.Decrypt()), _budget(f, out) if fac is f else None,
                        f.engine.op_counts(reset=True)["Relinarization"] if fac is f else None, out)
        assert np.array_equal(res["deferred"][0], res["default"][0])
        want = res["raw"][0]
        assert np.abs(np.asarray(res["raw"][3].Data)).max() < CRYPTONETS_PRIMES[0] * CRYPTONETS_PRIMES[1] / 2
        assert np.allclose(res["deferred"][0], want, rtol=1e-9, atol=1e-9 * np.abs(want).max())
        assert np.array_equal(np.argmax(res["deferred"][0], axis=1), np.argmax(want, axis=1))
        P = len(CRYPTONETS_PRIMES)
        assert res["default"][2] == P * 945 and res["deferred"][2] == P * 110, (res["default"][2], res["deferred"][2])
        assert res["deferred"][1] >= res["default"][1] - 1
        with capsys.disabled():
            print("\ncryptonets (%s): score noise budget %d bits default, %d bits deferred; relinearisations %d -> %d"
                  % (activation, res["default"][1], res["deferred"][1], res["default"][2], res["deferred"][2]))
    finally:
        f.Dispose()
