"""The FP64 accumulators of the diagonal product (k_diag_mac, k_diag_mac_resident) and of the summed tensor products
(k_behz_tensor_mac_fp) at coherent worst-case sums: every product of a sum is the same odd word of about p / 2, so a sum of more than 32
terms leaves the exact range of a double unless the kernel re-centres it (tests/fp64_accumulators.py builds the inputs and models the
sums).  49-bit coefficient primes, the widest the FP64 element-wise path takes.

Diagonal product: every output word equals the closed form S v w' at coefficient 0 (zero elsewhere), for B = 1, 2, 3, 5 and 9 clients
(CB = 1, 2, 4, 8) on two key slots in one call, streaming, partly and fully resident, groups of 116 to 128 diagonals (most not a multiple
of 8), N = 4096 and 8192, the folded product at two fold widths, and the integer path.  Each case pins the kernel by its ntt_info() and
the profiler's launches of the diagonal MAC (family 4, FP64 path only).

Summed tensor products: T = 8, 9, 33 and 255 identical terms on a 49-bit prime (K_c is unbounded there) and T = K_c = 256 on a 48-bit
one, against the oracle restatement, on the lazy FP64 inputs and the integer k_behz_tensor_mac."""
import numpy as np
import pytest

import fp64_accumulators as A
import worst_case_inputs as W

pytestmark = pytest.mark.gpu

T_PLAIN = 65537  # 1 mod 2N for N = 4096 and 8192
WEIGHT = T_PLAIN - 3  # -3: w' = q - 3, so v w' / p is as large as v and fmodmul's rounding error is at its widest
N1 = 64
ENV = ("CNHE_AUX_BASE", "CNHE_NTT_INT", "CNHE_KS_FUSED", "CNHE_MUL_FUSED")


def _engine(monkeypatch, t, N, q, dbc=10, env=None, seed=31):
    from cryptonets_b200.engine import Engine
    for var in ENV:
        monkeypatch.delenv(var, raising=False)
    for var, v in (env or {}).items():
        monkeypatch.setenv(var, v)
    eng = Engine([t], N, dbc, 20, -1, coeff_moduli=q)
    for var in ENV:
        monkeypatch.delenv(var, raising=False)
    assert eng.q == q
    eng.keygen(seed)
    return eng


@pytest.fixture(scope="module")
def mp():
    m = pytest.MonkeyPatch()
    yield m
    m.undo()


def _dropped(N):
    """(b, s) left out of the matrix: group g loses (5 g) mod 13 of its b = 1 diagonals, so the groups hold 116..128 terms"""
    out = set()
    for g in range(N // 2 // N1):
        for i in range(5 * g % 13):
            out.add((1, N1 * g + N1 - 1 - i))
    return out


class Ctx:
    def __init__(self, mp, N, env=None):
        self.N = N
        self.q = W.primes(49, N, 2)
        self.eng = _engine(mp, T_PLAIN, N, self.q, env=env)
        self.client = _engine(mp, T_PLAIN, N, self.q, env=env, seed=77)
        self.slot = self.eng.add_client_compact(self.client.save_compact_keys(public=False))
        self.w = [A.lift_weight(WEIGHT, T_PLAIN, p) for p in self.q]
        self.v = [[A.half_operand(p, w) for p, w in zip(self.q, self.w)], [A.widest_operand(p, w) for p, w in zip(self.q, self.w)]]

    def inputs(self, B):
        """B trivial constant ciphertexts: client b carries choice b % 2 and key slot 0 or the second client's, alternately"""
        out = []
        for b in range(B):
            x = self.eng.import_raw(A.trivial_ct(self.q, self.v[b % 2], self.N), 1, self.N, 1.0)
            if b % 2:
                x.set_key_slot(self.slot)
            out.append(x)
        return out

    def close(self):
        self.client.close()
        self.eng.close()


@pytest.fixture(scope="module")
def n4096(mp):
    c = Ctx(mp, 4096)
    dropped = _dropped(4096)
    M = A.diag_matrix(4096, WEIGHT - T_PLAIN, dropped)
    rows = [c.eng.plain(r, 1.0) for r in M]
    groups = A.diag_groups(4096, N1, dropped)
    c.lengths = [len(k) for _, k in groups]
    per_group = [n * c.eng.k * 4096 * 8 for n in c.lengths]
    c.mats = {"streaming": c.eng.diag_prepare(rows, N1, 0), "partly resident": c.eng.diag_prepare(rows, N1, sum(per_group[:3])),
              "resident": c.eng.diag_prepare(rows, N1, None)}
    c.eng.dispose_many(rows)
    yield c
    c.close()


def _served(eng, d, xs):
    """(outputs, launches of the FP64 diagonal MAC) of one mat_mul_diagonal call"""
    eng.prof_enable(True)
    eng.prof_collect()
    ys = eng.mat_mul_diagonal(d, xs)
    launches = eng.prof_collect()["scalar_mac_layer"]["launches"]
    eng.prof_enable(False)
    return ys, launches


def _check_diag(c, d, B, S, want_launches, closed=None):
    xs = c.inputs(B)
    ys, launches = _served(c.eng, d, xs)
    assert launches == want_launches
    for b, y in enumerate(ys):
        want = closed(b) if closed else A.diag_closed_form(c.q, c.v[b % 2], c.w, S, c.N)
        assert y.key_slot == (c.slot if b % 2 else 0)
        assert np.array_equal(y.export_raw(0, 0), want), b
    c.eng.dispose_many(xs + ys)


# mode: (resident giant steps, MAC launches: one wave of the resident prefix, one of the streamed groups)
MODES = {"streaming": (0, 1), "partly resident": (3, 2), "resident": (32, 1)}


@pytest.mark.parametrize("B", [1, 2, 3, 5, 9])
@pytest.mark.parametrize("mode", list(MODES))
def test_diagonal_product_at_coherent_sums(n4096, mode, B):
    c, d = n4096, n4096.mats[mode]
    info = d.info()
    assert (info["n1"], info["n2"], info["n_diags"]) == (N1, 32, sum(c.lengths))
    assert sorted(set(c.lengths)) == list(range(116, 129)) and min(c.lengths) >= 64
    assert d.ntt_info()["giant_steps"] == MODES[mode][0]
    _check_diag(c, d, B, sum(c.lengths), MODES[mode][1])


@pytest.mark.parametrize("mode", ["streaming", "resident"])
def test_diagonal_product_n8192(mp, mode):
    """N = 8192, every diagonal kept: 64 groups of 128 terms"""
    c = Ctx(mp, 8192)
    try:
        row = c.eng.plain(np.full(8192, float(WEIGHT - T_PLAIN)), 1.0)
        d = c.eng.diag_prepare([row] * 8192, N1, 0 if mode == "streaming" else None)
        assert d.info()["n_diags"] == 8192 and d.ntt_info()["giant_steps"] == (0 if mode == "streaming" else 64)
        _check_diag(c, d, 2, 8192, 1)
        d.dispose()
    finally:
        c.close()


@pytest.mark.parametrize("fold, mode", [(256, "streaming"), (2048, "resident")])
def test_folded_product_at_coherent_sums(n4096, fold, mode):
    """R = W rows of weight w over dim = N: W wrapped diagonals in groups of n1 = 64, the fold ladder doubling the sum up to N w v, then
    the mask of the first W slots -- the oracle's multiply_plain of the trivial constant N v w' by that mask"""
    from oracle.oracle_py import Oracle
    c = n4096
    orc = Oracle(T_PLAIN, c.N, -1, 10, 20, custom_q=c.q)
    row = c.eng.plain(np.full(c.N, float(WEIGHT - T_PLAIN)), 1.0)
    d = c.eng.diag_prepare([row] * fold, N1, 0 if mode == "streaming" else None, fold_width=fold)
    assert d.fold_width() == fold and d.info()["n_diags"] == fold
    assert d.ntt_info()["giant_steps"] == (0 if mode == "streaming" else fold // N1)
    mask = orc.encode(np.array([1] * fold + [0] * (c.N - fold), np.uint64))
    closed = {i: orc.multiply_plain(A.diag_closed_form(c.q, c.v[i], c.w, c.N, c.N), mask) for i in (0, 1)}
    _check_diag(c, d, 3, None, 1, closed=lambda b: closed[b % 2])
    d.dispose()
    c.eng.dispose_many([row])


def test_integer_fallback_gives_the_same_words(mp):
    """CNHE_NTT_INT: the dyadic products and additions, no FP64 MAC launch, the same closed-form words"""
    c = Ctx(mp, 4096, env={"CNHE_NTT_INT": "1"})
    try:
        dropped = _dropped(4096)
        M = A.diag_matrix(4096, WEIGHT - T_PLAIN, dropped)
        rows = [c.eng.plain(r, 1.0) for r in M]
        d = c.eng.diag_prepare(rows, N1, 0)
        c.eng.dispose_many(rows)
        _check_diag(c, d, 2, d.info()["n_diags"], 0)
        d.dispose()
    finally:
        c.close()


# ---------------------------------------------------------------- summed tensor products
# "q49": one 49-bit prime, whose Bsk leaves K_c unbounded (2^31 - 1); "kc": one 48-bit prime and a 26-bit plaintext prime, K_c = 256
TENSOR_CONTEXTS = {"q49": lambda N: W.primes(49, N, 1), "kc": lambda N: [_prime(48, N)]}
TENSOR_ENV = {"lazy": {}, "integer": {"CNHE_NTT_INT": "1"}}


def _prime(bits, N):
    from test_gpu_encrypted_product_deferred import _prime as p
    return p(bits, N)


@pytest.fixture(scope="module", params=[(c, e) for c in TENSOR_CONTEXTS for e in TENSOR_ENV], ids="-".join)
def tensor(mp, request):
    from oracle.oracle_py import Oracle
    name, path = request.param
    t, N = _prime(26, 4096), 4096
    eng = _engine(mp, t, N, TENSOR_CONTEXTS[name](N), dbc=16, env=TENSOR_ENV[path])
    orc = Oracle(t, N, -1, 16, 20, custom_q=eng.q)
    orc.keygen(31)
    # the FP64 element-wise path (and so k_behz_tensor_mac_fp) is on exactly when the diagonal MAC of a one-row matrix launches
    row = eng.plain(np.ones(4), 1.0)
    d = eng.diag_prepare([row])
    x = eng.encrypt(np.ones(4), 1.0)
    ys, launches = _served(eng, d, [x])
    assert launches == (0 if path == "integer" else 1)
    d.dispose()
    eng.dispose_many([row, x] + ys)
    yield eng, orc, name
    eng.close()


@pytest.mark.parametrize("T", [8, 9, 33, 255, "Kc"])
def test_summed_tensor_products_at_coherent_sums(tensor, T):
    """T identical terms: d0 gains (p - 3)/2, d1 p - 4 per term (tests/fp64_accumulators.py, tensor_operands), against the oracle
    restatement; T = K_c on the context where it is bounded"""
    from cryptonets_b200.engine import DENSE, SPARSE
    from test_gpu_encrypted_product_deferred import Restatement, kc_model
    eng, orc, name = tensor
    Kc = eng.product_sum_terms()
    assert Kc == kc_model(eng.q, eng.bsk, [orc.t], eng.N) == (256 if name == "kc" else 2 ** 31 - 1)
    if (T == "Kc") != (name == "kc"):
        pytest.skip("T = K_c runs on the kc context, the fixed T on q49")
    T = Kc if T == "Kc" else T
    q, N = eng.q, eng.N
    ops = [A.tensor_operands(p) for p in q]
    col_w = A.trivial_ct(q, [o[0][0] for o in ops], N, [o[0][1] for o in ops])
    sp_w = A.trivial_ct(q, [o[1][0] for o in ops], N, [o[1][1] for o in ops])
    col = eng.import_raw(col_w, 1, N, 1.0, DENSE)
    sparse = eng.import_raw(np.tile(sp_w, T), T, T, 1.0, SPARSE)
    out = eng.mat_mul_colmajor_sparse_deferred([col] * T, sparse)
    want = Restatement(orc).output([col_w] * T, [sp_w] * T, Kc)
    assert np.array_equal(out.export_raw(0, 0), want)
    eng.dispose_many([col, sparse, out])
