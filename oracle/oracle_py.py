"""ctypes binding of the CPU oracle (oracle/liboracle.so).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs.
The product package (cryptonets_b200/) never imports this module.
"""
import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
U64P = C.POINTER(C.c_uint64)


def build(force=False):
    so = os.path.join(_HERE, "liboracle.so")
    src = os.path.join(_HERE, "bfv_oracle.cpp")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(so):
            build()
        L = C.CDLL(so)
        L.orc_create.restype = C.c_void_p
        L.orc_create.argtypes = [C.c_uint64, C.c_uint32, C.c_int, C.c_int, C.c_int]
        L.orc_create_custom.restype = C.c_void_p
        L.orc_create_custom.argtypes = [C.c_uint64, C.c_uint32, U64P, C.c_int, C.c_int, C.c_int]
        L.orc_last_error.restype = C.c_char_p
        L.orc_minimal_primitive_root.restype = C.c_uint64
        L.orc_minimal_primitive_root.argtypes = [C.c_uint64, C.c_uint64]
        L.orc_t.restype = C.c_uint64
        L.orc_gamma.restype = C.c_uint64
        L.orc_N.restype = C.c_uint32
        L.orc_galois_elt_from_step.restype = C.c_uint64
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(U64P)


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


class Oracle:
    """One single-plain-modulus BFV context (== AtomicSealBfvEncryptedEnvironment, AtomicSealBfvVector.cs:19-206)."""

    def __init__(self, t, N, coeff_count=-1, dbc_relin=10, dbc_galois=20, custom_q=None):
        L = lib()
        if custom_q is not None:
            q = _u64(custom_q)
            self.h = L.orc_create_custom(C.c_uint64(t), N, _p(q), len(q), dbc_relin, dbc_galois)
        else:
            self.h = L.orc_create(C.c_uint64(t), N, coeff_count, dbc_relin, dbc_galois)
        if not self.h:
            raise ValueError(L.orc_last_error().decode())
        self.h = C.c_void_p(self.h)
        self.L = L
        self.N = N
        self.t = t
        self.k = L.orc_k(self.h)
        self.dbc_relin, self.dbc_galois = dbc_relin, dbc_galois
        q = np.zeros(self.k, np.uint64)
        L.orc_get_coeff_moduli(self.h, _p(q))
        self.q = [int(x) for x in q]
        b = np.zeros(self.k + 1, np.uint64)
        L.orc_get_bsk_moduli(self.h, _p(b))
        self.bsk = [int(x) for x in b]
        self.ct_words = 2 * self.k * N

    def __del__(self):
        try:
            self.L.orc_destroy(self.h)
        except Exception:
            pass

    def _chk(self, rc):
        if rc != 0:
            raise RuntimeError(self.L.orc_last_error().decode())

    def set_centered_mtilde(self, on):
        self.L.orc_set_centered_mtilde(self.h, int(on))

    # tables
    def ntt_tables(self, which):
        N = self.N
        w, ws, iw, iws = (np.zeros(N, np.uint64) for _ in range(4))
        inv_n = C.c_uint64()
        self.L.orc_get_ntt_tables(self.h, which, _p(w), _p(ws), _p(iw), _p(iws), C.byref(inv_n))
        return w, ws, iw, iws, inv_n.value

    def modulus_of(self, which):
        if which < self.k:
            return self.q[which]
        if which <= 2 * self.k:
            return self.bsk[which - self.k]
        return self.t

    def ntt(self, which, poly, inverse=False):
        a = _u64(poly).copy()
        (self.L.orc_ntt_inverse if inverse else self.L.orc_ntt_forward)(self.h, which, _p(a))
        return a

    def ntt_batch(self, which, polys, inverse=False, threads=1):
        a = _u64(polys).copy()
        self.L.orc_ntt_batch(self.h, which, _p(a), a.size // self.N, int(inverse), threads)
        return a

    # keys
    def keygen(self, seed):
        self.L.orc_keygen(self.h, C.c_uint64(seed))
        self.seed = seed

    def secret_key(self):
        a = np.zeros(self.k * self.N, np.uint64)
        self.L.orc_get_secret_key(self.h, _p(a))
        return a

    def public_key(self):
        a = np.zeros(2 * self.k * self.N, np.uint64)
        self.L.orc_get_public_key(self.h, _p(a))
        return a

    def relin_keys(self):
        n = self.L.orc_relin_key_count(self.h)
        a = np.zeros(n * self.ct_words, np.uint64)
        self.L.orc_get_relin_keys(self.h, _p(a))
        return a.reshape(n, 2, self.k, self.N)

    def galois_elts(self):
        n = self.L.orc_galois_elt_count(self.h)
        a = np.zeros(n, np.uint64)
        self.L.orc_get_galois_elts(self.h, _p(a))
        return [int(x) for x in a]

    def galois_key(self, elt):
        n = self.L.orc_galois_key_count(self.h)
        a = np.zeros(n * self.ct_words, np.uint64)
        self._chk(self.L.orc_get_galois_key(self.h, C.c_uint64(elt), _p(a)))
        return a.reshape(n, 2, self.k, self.N)

    def set_galois_key(self, elt, key):
        """Replaces the key of an element this context holds with `key` [count][2][k][N] (another key set's, e.g. a client key slot's)."""
        a = _u64(key).ravel()
        if a.size != self.L.orc_galois_key_count(self.h) * self.ct_words:
            raise ValueError("wrong Galois key size")
        self._chk(self.L.orc_set_galois_key(self.h, C.c_uint64(elt), _p(a)))

    # encoder
    def encode(self, values):
        v = _u64(values)
        out = np.zeros(self.N, np.uint64)
        self.L.orc_encode(self.h, _p(v), C.c_size_t(len(v)), _p(out))
        return out

    def decode(self, plain):
        p = _u64(plain)
        out = np.zeros(self.N, np.uint64)
        self.L.orc_decode(self.h, _p(p), _p(out))
        return out

    # encrypt / decrypt
    def encrypt(self, plain, nonce):
        p = _u64(plain)
        out = np.zeros(self.ct_words, np.uint64)
        self.L.orc_encrypt(self.h, _p(p), C.c_size_t(len(p)), C.c_uint64(nonce), _p(out))
        return out

    def decrypt(self, ct):
        ct = _u64(ct).ravel()
        size = ct.size // (self.k * self.N)
        out = np.zeros(self.N, np.uint64)
        self._chk(self.L.orc_decrypt(self.h, _p(ct), size, _p(out)))
        return out

    def noise_budget(self, ct):
        ct = _u64(ct).ravel()
        return self.L.orc_noise_budget(self.h, _p(ct), ct.size // (self.k * self.N))

    # evaluator
    def _bin(self, fn, a, b):
        a, b = _u64(a).ravel(), _u64(b).ravel()
        out = np.zeros_like(a)
        fn(self.h, _p(a), _p(b), a.size // (self.k * self.N), _p(out))
        return out

    def add(self, a, b):
        return self._bin(self.L.orc_add, a, b)

    def sub(self, a, b):
        return self._bin(self.L.orc_sub, a, b)

    def negate(self, a):
        a = _u64(a).ravel()
        out = np.zeros_like(a)
        self.L.orc_negate(self.h, _p(a), a.size // (self.k * self.N), _p(out))
        return out

    def add_plain(self, ct, plain, sub=False):
        ct, p = _u64(ct).ravel(), _u64(plain)
        out = np.zeros_like(ct)
        (self.L.orc_sub_plain if sub else self.L.orc_add_plain)(
            self.h, _p(ct), ct.size // (self.k * self.N), _p(p), C.c_size_t(len(p)), _p(out))
        return out

    def multiply_plain(self, ct, plain):
        ct, p = _u64(ct).ravel(), _u64(plain)
        out = np.zeros_like(ct)
        self._chk(self.L.orc_multiply_plain(self.h, _p(ct), ct.size // (self.k * self.N), _p(p), C.c_size_t(len(p)), _p(out)))
        return out

    def multiply(self, a, b):
        a, b = _u64(a).ravel(), _u64(b).ravel()
        out = np.zeros(3 * self.k * self.N, np.uint64)
        self._chk(self.L.orc_multiply(self.h, _p(a), _p(b), _p(out)))
        return out

    def relinearize(self, ct3):
        ct3 = _u64(ct3).ravel()
        out = np.zeros(self.ct_words, np.uint64)
        self._chk(self.L.orc_relinearize(self.h, _p(ct3), _p(out)))
        return out

    def apply_galois(self, ct, elt):
        ct = _u64(ct).ravel()
        out = np.zeros_like(ct)
        self._chk(self.L.orc_apply_galois(self.h, _p(ct), C.c_uint64(elt), _p(out)))
        return out

    def rotate_rows(self, ct, steps):
        ct = _u64(ct).ravel()
        out = np.zeros_like(ct)
        self._chk(self.L.orc_rotate_rows(self.h, _p(ct), int(steps), _p(out)))
        return out

    def rotate_columns(self, ct):
        ct = _u64(ct).ravel()
        out = np.zeros_like(ct)
        self._chk(self.L.orc_rotate_columns(self.h, _p(ct), _p(out)))
        return out

    def galois_elt_from_step(self, steps):
        return int(self.L.orc_galois_elt_from_step(self.h, int(steps)))

    def behz_lift(self, poly_q):
        a = _u64(poly_q).ravel()
        out = np.zeros((self.k + 1) * self.N, np.uint64)
        self._chk(self.L.orc_behz_lift(self.h, _p(a), _p(out)))
        return out

    def behz_floor(self, poly_q_bsk):
        a = _u64(poly_q_bsk).ravel()
        out = np.zeros(self.k * self.N, np.uint64)
        self._chk(self.L.orc_behz_floor(self.h, _p(a), _p(out)))
        return out

    # layer drivers (CPU baseline)
    def mac_layer(self, in_cts, gather, weights, bias, M, K, threads=1, m_begin=0, m_step=1, out=None):
        in_cts = _u64(in_cts).ravel()
        n_in = in_cts.size // self.ct_words
        g = None if gather is None else np.ascontiguousarray(gather, dtype=np.int32)
        w = _u64(weights).ravel()
        b = None if bias is None else _u64(bias).ravel()
        if out is None:
            out = np.zeros(M * self.ct_words, np.uint64)
        self._chk(self.L.orc_mac_layer(
            self.h, _p(in_cts), n_in, None if g is None else g.ctypes.data_as(C.POINTER(C.c_int32)), _p(w),
            None if b is None else _p(b), M, K, _p(out), threads, m_begin, m_step))
        return out

    def square_layer(self, in_cts, threads=1, begin=0, step=1, out=None):
        in_cts = _u64(in_cts).ravel()
        n = in_cts.size // self.ct_words
        if out is None:
            out = np.zeros_like(in_cts)
        self._chk(self.L.orc_square_layer(self.h, _p(in_cts), n, _p(out), threads, begin, step))
        return out
