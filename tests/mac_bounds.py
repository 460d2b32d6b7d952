"""The scalar-MAC layer's accumulator bounds as exact integers, the words that reach them, and a closed form of the layer.

`mac_channel` (csrc/vec.cu) serves each plaintext channel of a layer with the first of four kernels whose bound holds:
  umma    wgmma on slab inputs: int32 limb sums of s8 x u8 products, total_chunks * 32 * 127 * 255 < 2^31, plan fits in shared memory
  imma    mma.sync on one gather row: W1 and W2 limb sums in one int32 accumulator, K * 254 * 255 < 2^31
  fp64    sums of w * x_lo in doubles, x cut into 26-bit halves: |w| < 2^17 and K * wmax * 2^26 < 2^52
  int128  128-bit sums of lifted weights x words: 2 * maxbits + bits(K) <= 127, a wider layer is refused
The predicates below restate those gates; the words below are the ones that drive each accumulator to its bound.  The closed form sums
each output's weights per distinct input first, so a layer that reads one input 33155 times costs one product per word.

No GPU is needed here: tests/test_mac_bounds_model.py checks this module against brute force and the CPU oracle, and
tests/test_gpu_mac_bounds.py runs the kernels on these operands."""
import numpy as np

import worst_case_inputs as W

TWO31 = 1 << 31
TWO52 = 1 << 52
FP64_SPLIT = 26      # bits in the low half of a word on the FP64 path
W_BYTE = 254         # largest merged weight the tensor-core kernels take (W1 + W2, each a signed byte clamped to +-127)


def limbs(maxbits):
    return (maxbits + 7) // 8


def primes(bits, N, count=1):
    """the `count` largest `bits`-bit primes = 1 mod 2N (at most 50 bits here: none is gamma, m_sk or a SEAL auxiliary prime, all 61 bits)"""
    out, c = [], ((1 << bits) - 1) // (2 * N) * (2 * N) + 1
    while len(out) < count:
        if W.is_prime(c):
            out.append(c)
        c -= 2 * N
    assert all(p.bit_length() == bits for p in out)
    return out


def _largest_with_low_ones(q, low_bits):
    """the largest word below q whose low `low_bits` bits are all ones"""
    low = (1 << low_bits) - 1
    return (q - 1 - low) >> low_bits << low_bits | low


def maximal_limb_word(q, maxbits):
    """the largest word below q whose lower L - 1 bytes are all 0xff (L = limbs(maxbits)): every limb but the top one at 255"""
    return _largest_with_low_ones(q, 8 * (limbs(maxbits) - 1))


def maximal_low_half_word(q):
    """the largest word below q whose low 26 bits are all ones: the FP64 path's x_lo at 2^26 - 1"""
    return _largest_with_low_ones(q, FP64_SPLIT)


# ---------------------------------------------------------------- the gates (csrc/vec.cu: mac_route, mac_umma_plan, mac_prepare)
def imma_admits(K):
    return K >= 32 and K * 2 * 127 * 255 < TWO31


def fp64_admits(K, wmax, maxbits):
    return maxbits <= 50 and wmax < 1 << 17 and K * wmax << FP64_SPLIT < TWO52


def int128_admits(K, maxbits):
    return 2 * maxbits + K.bit_length() <= 127


def umma_chunks_admitted(total_chunks):
    return total_chunks * 32 * 127 * 255 < TWO31


def largest(pred, lo=1):
    """the largest K >= lo with pred(K), for a predicate that holds up to some K and fails beyond it"""
    assert pred(lo)
    hi = lo
    while pred(hi * 2):
        hi *= 2
    step = hi
    while step:
        if pred(hi + step):
            hi += step
        step //= 2
    return hi


def umma_plan(gather, w, limbs_=6):
    """the wgmma planner's verdict on a layer (cnhe_debug_mac_plan, host code only): None when no plan fits, else its bundles, chunks per
    tile, weight bytes and W2 taps"""
    import ctypes as C
    from cryptonets_b200 import _lib
    fn = _lib.lib().cnhe_debug_mac_plan
    fn.restype = C.c_int
    fn.argtypes = [C.POINTER(C.c_int32), C.POINTER(C.c_double), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
    g = np.ascontiguousarray(gather, dtype=np.int32)
    ww = np.ascontiguousarray(w, dtype=np.float64)
    out = (C.c_int * 4)()
    ok = fn(g.ctypes.data_as(C.POINTER(C.c_int32)), ww.ctypes.data_as(C.POINTER(C.c_double)), g.shape[0], g.shape[1], limbs_, out)
    return None if not ok else dict(bundles=out[0], chunks=out[1], weight_bytes=out[2], extra_taps=out[3])


def wide_dense(M, K):
    """a dense layer over inputs 0..K-1 whose weights are all +254 (even outputs) or -254 (odd ones): every tap needs a W2 column"""
    gather = np.tile(np.arange(K, dtype=np.int32), (M, 1))
    w = np.where(np.arange(M)[:, None] % 2 == 0, W_BYTE, -W_BYTE) * np.ones((M, K), dtype=np.int64)
    return gather, w


def widest_umma_window(limbs_, M=16):
    """the largest K (a whole number of 32-tap chunks) whose all-+-254 dense layer the wgmma planner fits in shared memory"""
    c = largest(lambda c: umma_plan(*wide_dense(M, 32 * c), limbs_) is not None)
    return 32 * c


def route(K, M, maxbits, wmax, rows=1, planned=False):
    """the kernel mac_channel picks for a channel: rows = distinct gather rows, planned = the wgmma planner found a plan that fits"""
    L = limbs(maxbits)
    if planned and M >= 8 and maxbits <= 50 and 5 <= L <= 7 and wmax <= W_BYTE:
        return "umma"
    if rows == 1 and wmax <= W_BYTE and M >= 8 and maxbits <= 50 and 5 <= L <= 7 and imma_admits(K):
        return "imma"
    if fp64_admits(K, wmax, maxbits):
        return "fp64"
    return "int128" if int128_admits(K, maxbits) else None


# ---------------------------------------------------------------- the layer in closed form
def delta(q, t):
    Q = 1
    for p in q:
        Q *= p
    return Q // t


def merged(gather, w, n_in):
    """[M][n_in] int64: per output, the sum of its weights over every tap that reads input j (padded taps, -1, carry nothing)"""
    g, ww = np.asarray(gather), np.asarray(w, dtype=np.int64)
    out = np.zeros((g.shape[0], n_in), dtype=np.int64)
    for m in range(g.shape[0]):
        live = g[m] >= 0
        np.add.at(out[m], g[m][live], ww[m][live])
    return out


def mac_closed_form(words, gather, w, bias, q, t):
    """out[m] = sum_j (sum_{k: gather[m, k] = j} w[m, k]) x_j mod q_l, plus Delta b[m] on coefficient 0 of c0.

    words [n_in][polys][k][N] canonical residues of one plaintext channel; gather [M][K] (-1: padded tap); w [M][K] the signed (centred)
    weights, which is the lift SEAL gives a plaintext scalar; bias [M] signed constants or None.  Returns [M][polys][k][N] uint64.
    The sums are exact: each word is cut into 25-bit halves, summed in int64 and joined in Python integers."""
    x = np.asarray(words, dtype=np.uint64)
    n_in, shape = x.shape[0], x.shape[1:]
    Wm = merged(gather, w, n_in)
    assert int(np.abs(Wm).sum(axis=1).max()) * max(1 << 25, max(q) >> 25) < 1 << 63
    xs = x.reshape(n_in, -1)
    lo = Wm @ (xs & np.uint64((1 << 25) - 1)).astype(np.int64)
    hi = Wm @ (xs >> np.uint64(25)).astype(np.int64)
    qo = np.array(q, dtype=object)[None, None, :, None]
    r = (hi.astype(object) * (1 << 25) + lo.astype(object)).reshape((-1,) + shape) % qo
    if bias is not None:
        dl = delta(q, t)
        for m in range(r.shape[0]):
            for l, p in enumerate(q):
                r[m, 0, l, 0] = (r[m, 0, l, 0] + dl * int(bias[m])) % p
    return r.astype(np.uint64)


def centred(v, t):
    """integers as signed residues mod t in (-t/2, t/2]: the weight a plaintext scalar carries"""
    r = np.asarray(v, dtype=np.int64) % t
    return np.where(r > t // 2, r - t, r)


def residues(v, t):
    """signed integers as residues mod t (what the oracle takes)"""
    v = np.asarray(v, dtype=np.int64)
    return np.where(v < 0, v + t, v).astype(np.uint64)
