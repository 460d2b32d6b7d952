"""cnhe_mat_mul_colmajor_sparse_deferred: encrypted columns times an encrypted sparse vector, the tensor products summed in the NTT domain,
one BEHZ floor per chunk of at most K_c terms and one relinearisation per output block.

Every output word must equal the CPU oracle's restatement, per plaintext prime and output block i:
    Y_i = sum over chunks (mod q) of floor(INTT(sum_{k in chunk} NTT(lift(cols[k]_i)) * NTT(lift(sparse_k)))),   out_i = relinearize(Y_i)
with the oracle's own lift, transforms, floor and relinearisation, on the lazy FP64, canonical FP64 (CNHE_NO_LAZY) and integer
(CNHE_NTT_INT, 53/56-bit moduli) paths, both m~ conventions, fast and SEAL Bsk, N = 4096 / 8192 / 16384, both key-switch paths.  K_c is
checked against its derivation and pinned at the bound with constructed operands; the output decrypts to the existing call's values, the
operation counts are the documented ones and every refusal leaves the output NULL."""
import ctypes as C

import numpy as np
import pytest

from cryptonets_b200._lib import CnheError

pytestmark = pytest.mark.gpu

ERR_INVALID = -1
M_TILDE = 1 << 32


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


# "kc": one 48-bit coefficient prime and a 26-bit plaintext prime leave the fast Bsk (two 48-bit primes) so little room that K_c = 256
CONTEXTS = {
    "n4096": dict(t=[40961], N=4096, dbc=10, q=None),
    "kc": dict(t=[_prime(26, 4096)], N=4096, dbc=16, q=[_prime(48, 4096)]),
    "n8192-cryptonets": dict(t=[549764251649, 549764284417], N=8192, dbc=10, q=None),
    "n16384": dict(t=[786433], N=16384, dbc=60, q=None),
    "n4096-q53": dict(t=[40961], N=4096, dbc=10, q=[_prime(53, 4096), _prime(56, 4096)]),
}
ENV = ("CNHE_AUX_BASE", "CNHE_NO_LAZY", "CNHE_NTT_INT", "CNHE_KS_FUSED", "CNHE_MUL_FUSED")


def _pair(name, monkeypatch, env=None):
    from cryptonets_b200.engine import Engine
    from oracle.oracle_py import Oracle
    cfg = CONTEXTS[name]
    for var in ENV:
        monkeypatch.delenv(var, raising=False)
    for var, v in (env or {}).items():
        monkeypatch.setenv(var, v)
    eng = Engine(cfg["t"], cfg["N"], cfg["dbc"], 20, -1, coeff_moduli=cfg["q"])
    eng.keygen(31)
    orcs = []
    for ch, t in enumerate(cfg["t"]):
        o = Oracle(t, cfg["N"], -1, cfg["dbc"], 20, custom_q=cfg["q"])
        o.keygen(31 + ch)
        orcs.append(o)
    return eng, orcs


def kc_model(q, bsk, t, N):
    """K_c as DESIGN 4.14 derives it: the largest K with 2 K N t Q (1 + k/m~)^2 + k + 1 < B ((m_sk - 1)/2 - na), clamped to [1, 2^31 - 1]"""
    k, na, msk = len(q), len(bsk) - 1, bsk[-1]
    B = Q = 1
    for b in bsk[:-1]:
        B *= b
    for x in q:
        Q *= x
    limit = (B * ((msk - 1) // 2 - na) - k - 1) * M_TILDE * M_TILDE
    per = 2 * N * max(t) * Q * (M_TILDE + k) ** 2
    return max(1, min((limit - 1) // per, 2 ** 31 - 1))


class Restatement:
    """the oracle's composition, with each ciphertext lifted and transformed once (cached by its words)"""

    def __init__(self, orc):
        self.orc, self.cache = orc, {}
        self.mods = [orc.modulus_of(w) for w in range(2 * orc.k + 1)]

    def lifted(self, ct):
        key = ct.tobytes()
        if key not in self.cache:
            orc, k, N = self.orc, self.orc.k, self.orc.N
            ct = ct.reshape(2, k, N)
            polys = []
            for p in range(2):
                res = np.concatenate([ct[p].reshape(-1), orc.behz_lift(ct[p])]).reshape(2 * k + 1, N)
                polys.append(np.stack([orc.ntt(w, res[w]) for w in range(2 * k + 1)]))
            self.cache[key] = np.stack(polys)
        return self.cache[key]

    def floor_sum(self, pairs):
        """floor_BEHZ(t INTT(sum of the tensor products of the (a, b) ciphertext pairs)), size 3"""
        orc, N = self.orc, self.orc.N
        A = np.stack([self.lifted(a) for a, _ in pairs]).astype(object)
        B = np.stack([self.lifted(b) for _, b in pairs]).astype(object)
        out = []
        for part in range(3):
            res = []
            for w, m in enumerate(self.mods):
                if part == 0:
                    s = (A[:, 0, w] * B[:, 0, w]).sum(axis=0)
                elif part == 1:
                    s = (A[:, 0, w] * B[:, 1, w] + A[:, 1, w] * B[:, 0, w]).sum(axis=0)
                else:
                    s = (A[:, 1, w] * B[:, 1, w]).sum(axis=0)
                res.append(orc.ntt(w, (s % m).astype(np.uint64), inverse=True).astype(object) * (orc.t % m) % m)  # times t, as orc_multiply
            out.append(orc.behz_floor(np.concatenate(res).astype(np.uint64)))
        return np.concatenate(out)

    def output(self, cols, sparse, Kc):
        Y = None
        for j0 in range(0, len(cols), Kc):
            f = self.floor_sum(list(zip(cols[j0:j0 + Kc], sparse[j0:j0 + Kc])))
            Y = f if Y is None else self.orc.add(Y, f)
        return self.orc.relinearize(Y)


def _operands(eng, K, blocks, seed, dim=None):
    from cryptonets_b200.engine import DENSE, SPARSE
    rng = np.random.default_rng(seed)
    dim = dim or blocks * eng.N - 3
    cols = [eng.encrypt(rng.integers(-60, 60, dim).astype(np.float64), 1.0, DENSE) for _ in range(K)]
    sparse = eng.encrypt(rng.integers(-60, 60, K).astype(np.float64), 1.0, SPARSE)
    return cols, sparse


def _check(eng, orcs, cols, sparse, out, blocks=None, mtilde=False):
    Kc = eng.product_sum_terms()
    K = len(cols)
    for ch, orc in enumerate(orcs):
        orc.set_centered_mtilde(mtilde)
        R = Restatement(orc)
        s = [sparse.export_raw(ch, j) for j in range(K)]
        for i in (range(cols[0].blocks) if blocks is None else blocks):
            want = R.output([c.export_raw(ch, i) for c in cols], s, Kc)
            assert np.array_equal(out.export_raw(ch, i), want), (ch, i)


CASES = [  # (context, env, [(K, blocks)], m~ conventions)
    ("n4096", {}, [(1, 1), (2, 3), (100, 1)], (False, True)),
    ("n4096", {"CNHE_AUX_BASE": "seal"}, [(2, 3), (100, 1)], (False, True)),
    ("n4096", {"CNHE_NO_LAZY": "1"}, [(2, 3), (30, 1)], (False,)),
    ("n4096", {"CNHE_NTT_INT": "1"}, [(2, 3), (30, 1)], (False, True)),
    ("n4096-q53", {}, [(2, 3), (30, 1)], (False,)),
    ("kc", {}, [(2, 1), ("Kc", 1), ("Kc+1", 1)], (False, True)),
    ("n8192-cryptonets", {}, [(2, 1), (100, 1)], (False,)),
    ("n16384", {}, [(1, 1), (3, 1)], (False,)),
]


@pytest.mark.parametrize("case", range(len(CASES)), ids=["%s-%s" % (c[0], "-".join(c[1].values()) or "lazy") for c in CASES])
def test_words_equal_oracle_restatement(case, monkeypatch):
    """both key-switch paths (forced: the outputs here are fewer than 64) on every product path and m~ convention"""
    name, env, shapes, conventions = CASES[case]
    eng, orcs = _pair(name, monkeypatch, env)
    try:
        Kc = eng.product_sum_terms()
        assert Kc == kc_model([int(x) for x in eng.q], eng.bsk, CONTEXTS[name]["t"], eng.N)
        if name == "kc":
            assert Kc == 256
        for K, blocks in shapes:
            K = {"Kc": Kc, "Kc+1": Kc + 1}.get(K, K)
            cols, sparse = _operands(eng, K, blocks, K + blocks)
            for mt in conventions:
                eng.set_option("behz_centered_mtilde", int(mt))
                for fused in ("1", "0"):
                    monkeypatch.setenv("CNHE_KS_FUSED", fused)
                    out = eng.mat_mul_colmajor_sparse_deferred(cols, sparse)
                    assert out.blocks == blocks and out.dim == cols[0].dim and out.scale == 1.0
                    _check(eng, orcs, cols, sparse, out, mtilde=mt)
                    out.dispose()
            for v in cols + [sparse]:
                v.dispose()
    finally:
        eng.close()


def test_fused_key_switch_at_64_outputs(monkeypatch):
    """65 output blocks: the default key-switch path is the fused kernel; blocks 0, 33 and 64 against the restatement"""
    eng, orcs = _pair("n4096", monkeypatch)
    try:
        cols, sparse = _operands(eng, 2, 65, 3)
        out = eng.mat_mul_colmajor_sparse_deferred(cols, sparse)
        _check(eng, orcs, cols, sparse, out, blocks=(0, 33, 64))
    finally:
        eng.close()


def test_exact_at_the_bound(monkeypatch):
    """K_c terms of maximal magnitude in one chunk: every column block and sparse element has all coefficients q - 1, which lifts to
    Q - 1 with the uncentred m~, so every coefficient of the sum reaches 2 K_c N (Q - 1)^2 in d1 -- the bound K_c is derived from.  The
    oracle's floor of the sum (its SEAL Bsk is exact far beyond K_c) is within k + 1 of the exact round(t X / Q) of textbook_bfv, and the
    GPU output equals its relinearisation word for word, so the context's own Bsk floored the sum exactly."""
    from cryptonets_b200.engine import DENSE, SPARSE
    from oracle.textbook_bfv import round_div
    eng, orcs = _pair("kc", monkeypatch)
    try:
        orc, N, Kc = orcs[0], eng.N, eng.product_sum_terms()
        Q, t, k = orc.q[0], orc.t, orc.k
        word = np.full(eng.ct_words, Q - 1, np.uint64)
        col = eng.import_raw(word, 1, N, 1.0, DENSE)
        sparse = eng.import_raw(np.tile(word, Kc), Kc, Kc, 1.0, SPARSE)
        out = eng.mat_mul_colmajor_sparse_deferred([col] * Kc, sparse)
        R = Restatement(orc)
        Y = R.floor_sum([(word, word)] * Kc).reshape(3, N)
        j = np.arange(N, dtype=object)
        base = Kc * (Q - 1) ** 2 * (2 * j + 2 - N)  # negacyclic product of two all-(Q-1) polynomials, summed K_c times
        for part, mult in enumerate((1, 2, 1)):
            X = base * mult
            assert max(abs(int(x)) for x in X) >= 2 * (Kc - 1) * N * (Q - 1) ** 2 if part == 1 else True
            exact = np.array([round_div(t * int(x), Q) % Q for x in X], dtype=object)
            diff = (Y[part].astype(object) - exact) % Q
            diff = np.where(diff > Q // 2, diff - Q, diff)
            assert max(abs(int(d)) for d in diff) <= k + 1, part
        assert np.array_equal(out.export_raw(0, 0), orc.relinearize(Y.reshape(-1)))
    finally:
        eng.close()


def test_decrypts_to_the_existing_call(monkeypatch, capsys):
    """CryptoNets parameters, two blocks: the deferred output decrypts to cnhe_mat_mul_colmajor_sparse's values and keeps at least its
    noise budget"""
    eng, _ = _pair("n8192-cryptonets", monkeypatch)
    try:
        cols, sparse = _operands(eng, 40, 2, 11)
        old = eng.mat_mul_colmajor_sparse(cols, sparse)
        new = eng.mat_mul_colmajor_sparse_deferred(cols, sparse)
        assert new.dim == old.dim and new.scale == old.scale and new.blocks == old.blocks
        assert np.array_equal(eng.decrypt(new), eng.decrypt(old))
        b_old = min(eng.noise_budget(old, ch, b) for ch in range(eng.P) for b in range(old.blocks))
        b_new = min(eng.noise_budget(new, ch, b) for ch in range(eng.P) for b in range(new.blocks))
        assert b_new >= b_old
        with capsys.disabled():
            print("\nK = 40, 2 blocks, N = 8192: noise budget %d bits existing, %d bits deferred" % (b_old, b_new))
    finally:
        eng.close()


def test_operation_counts(monkeypatch):
    """K bl Multiply, bl (K - 1) Addition, bl Relinearize and K bl AddMany items per plaintext prime"""
    eng, _ = _pair("n8192-cryptonets", monkeypatch)
    try:
        K, bl, P = 7, 2, eng.P
        cols, sparse = _operands(eng, K, bl, 5)
        eng.op_counts(reset=True)
        eng.mat_mul_colmajor_sparse_deferred(cols, sparse)
        got = {k: v for k, v in eng.op_counts(reset=True).items() if v}
        assert got == {"Multiplication": P * K * bl, "Addition": P * bl * (K - 1), "Relinarization": P * bl, "AddManyItemCount": P * K * bl}, got
    finally:
        eng.close()


def _raw_call(eng, cols, sparse):
    from cryptonets_b200._lib import VECP
    out = VECP()
    rc = eng.L.cnhe_mat_mul_colmajor_sparse_deferred(eng.h, (VECP * len(cols))(*[v.h for v in cols]), len(cols), sparse.h, C.byref(out))
    return rc, out


def test_refusals(monkeypatch):
    from cryptonets_b200.engine import DENSE, SPARSE
    eng, _ = _pair("n4096", monkeypatch)
    try:
        N = eng.N
        cols, sparse = _operands(eng, 3, 1, 8)
        other = _operands(eng, 3, 1, 9)[1]
        other.set_key_slot(eng.add_client_compact(eng.save_compact_keys(public=False)))
        # the same column listed over and over: a chunk whose lifted operands alone pass 8 GiB (K_c is far larger here)
        kt = eng.k + eng.kb
        huge = 2 ** 30 // (2 * 2 * kt * N) + 1
        cases = {
            "mixed key slots": (cols, other),
            "plain sparse vector": (cols, eng.plain(np.ones(3), 1.0, SPARSE)),
            "plain columns": ([eng.plain(np.ones(N), 1.0, DENSE)] * 3, sparse),
            "dimension mismatch": (cols[:2], sparse),
            "dense vector argument": (cols, eng.encrypt(np.ones(3), 1.0, DENSE)),
            "columns of two dimensions": (cols[:2] + [eng.encrypt(np.ones(N + 5), 1.0, DENSE)], sparse),
            "chunk beyond 8 GiB": ([cols[0]] * huge, eng.import_raw(np.tile(sparse.export_raw(0, 0), huge), huge, huge, 1.0, SPARSE)),
        }
        for what, (cs, sp) in cases.items():
            rc, out = _raw_call(eng, cs, sp)
            assert rc == ERR_INVALID, what
            assert not out, what
        with pytest.raises(CnheError, match="cnhe_mat_mul_colmajor_sparse"):
            eng.mat_mul_colmajor_sparse_deferred([eng.plain(np.ones(N), 1.0, DENSE)] * 3, sparse)
        assert eng.mat_mul_colmajor_sparse_deferred(cols, sparse).dim == cols[0].dim
    finally:
        eng.close()


def test_matrix_mul_keyword():
    """B200BfvMatrix.Mul(DeferRelinearization=True) decrypts to Mul's values; elsewhere the keyword raises"""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.interfaces import EMatrixFormat, EVectorFormat
    f = B200BfvFactory([40961], 4096, seed=3)
    try:
        rng = np.random.default_rng(4)
        m = rng.integers(-20, 20, (50, 6)).astype(np.float64)
        v = rng.integers(-20, 20, 6).astype(np.float64)
        M = f.GetEncryptedMatrix(m, EMatrixFormat.ColumnMajor, 1.0)
        V = f.GetEncryptedVector(v, EVectorFormat.sparse, 1.0)
        want = np.asarray(M.Mul(V).Decrypt())
        assert np.array_equal(np.asarray(M.Mul(V, DeferRelinearization=True).Decrypt()), want)
        assert np.array_equal(want, m @ v)
        with pytest.raises(Exception, match="DeferRelinearization"):
            M.Mul(f.GetPlainVector(v, EVectorFormat.sparse, 1.0), DeferRelinearization=True)
        with pytest.raises(Exception, match="DeferRelinearization"):
            f.GetEncryptedMatrix(m.T, EMatrixFormat.RowMajor, 1.0).Mul(f.GetEncryptedVector(v, EVectorFormat.dense, 1.0), DeferRelinearization=True)
    finally:
        f.Dispose()
