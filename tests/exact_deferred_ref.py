"""Exact CPU reference of a scalar-MAC layer over unrelinearised size-3 products (DESIGN 4.15).

Relinearising (c0, c1, c2) adds INTT(sum_d NTT(digit_d(c2)) * K_d) to (c0, c1), and both the key switch and the layer are linear modulo
each q_l, so output m of the layer over the relinearised products is the closed form

    (sum_j W_mj (c0_j, c1_j) + Delta bias_m on c0) mod q_l  +  INTT(sum_d NTT(S_md mod q_l) * K_d),   S_md = sum_j W_mj digit_d(c2_j)

with W_mj the weights centred modulo t (as multiply_plain reads a plaintext scalar) and the digits cut by worst_case_inputs.digit_map.
Every value here is an exact integer: S_md in int64 (asserted below 2^62), the linear part from 25-bit halves of the words.  No GPU is
needed; tests/test_exact_deferred_ref.py checks this form against the oracle's relinearise + scalar MAC, and
tests/test_gpu_exact_deferred_edges.py holds the GPU's exact path to it."""
import numpy as np

import worst_case_inputs as W


def centred_weights(w, t):
    """residues mod t (M x K) -> signed integers in (-t/2, t/2], what the layer multiplies by"""
    w = np.asarray(w, dtype=np.int64)
    return np.where(w >= (t + 1) // 2, w - t, w)


def maximal_word(q, w):
    """the largest word below q whose digits below the top one are all 2^w - 1"""
    top = (q.bit_length() - 1) // w * w
    low = (1 << top) - 1
    return (q - 1 - low) >> top << top | low


def maximal_c2(q, w, N):
    """(k x N) c2 residues of maximal words"""
    return np.array([[maximal_word(p, w)] * N for p in q], dtype=np.uint64)


def edge_weights(total, wmax=254):
    """magnitudes <= wmax, as many at wmax as fit, summing to total: the fewest taps that reach a given sum of |W|"""
    return [wmax] * (total // wmax) + ([total % wmax] if total % wmax else [])


def bound_edge(w):
    """the largest sum of |W| the exact path takes at digit width w on moduli of 32 bits or more: sum * (2^w - 1) < 2^31"""
    return ((1 << 31) - 1) // ((1 << w) - 1)


def _taps(gather, m, K):
    """(input index, tap index) of output m's taps that are not padded"""
    row = np.arange(K) if gather is None else np.asarray(gather[m])
    kk = np.nonzero(row >= 0)[0]
    return row[kk].astype(np.int64), kk


def digit_sums(cts3, wc, gather, q, w, m):
    """S_m (D x N, int64): S_md = sum_j W_mj digit_d(c2_j) over output m's taps, cts3 (n_in x 3 x k x N), wc centred weights (M x K)"""
    idx, kk = _taps(gather, m, wc.shape[1])
    wm = wc[m, kk]
    assert int(np.abs(wm).sum()) * ((1 << w) - 1) < 1 << 62
    mask = np.uint64((1 << w) - 1)
    c2 = cts3[idx, 2]
    return np.stack([wm @ ((c2[:, i, :] >> np.uint64(sh)) & mask).astype(np.int64) for i, sh in W.digit_map(q, w)])


def linear_part(cts3, wc, gather, q, m):
    """(2 x k x N) sum_j W_mj (c0_j, c1_j) mod q_l, from the 25-bit halves of the words (each half-sum exact in int64)"""
    idx, kk = _taps(gather, m, wc.shape[1])
    wm = wc[m, kk]
    assert int(np.abs(wm).sum()) < 1 << 38
    k, N = len(q), cts3.shape[-1]
    out = np.zeros((2, k, N), np.uint64)
    for p in range(2):
        for l, ql in enumerate(q):
            x = cts3[idx, p, l]
            lo = wm @ (x & np.uint64((1 << 25) - 1)).astype(np.int64)
            hi = wm @ (x >> np.uint64(25)).astype(np.int64)
            out[p, l] = ((hi.astype(object) * (1 << 25) + lo.astype(object)) % ql).astype(np.uint64)
    return out


def bias_words(orc, values):
    """(k x N) words a bias of slot values (residues mod t) adds to c0: the oracle's add_plain on a zero ciphertext"""
    zero = np.zeros(orc.ct_words, np.uint64)
    return orc.add_plain(zero, orc.encode(np.asarray(values, dtype=np.uint64))).reshape(2, orc.k, orc.N)[0]


def closed_form(orc, cts3, wc, gather, keys, w, m, bias=None):
    """(2 x k x N) words of output m: cts3 (n_in x 3 x k x N) canonical size-3 products, wc centred weights (M x K), gather (M x K,
    -1 padded) or None (tap k is input k), keys the NTT-domain relinearisation keys (D x 2 x k x N), bias None or the (k x N) words of
    bias_words.  orc: an Oracle of the context's q and N (its transforms)"""
    q = orc.q
    cts3 = np.asarray(cts3, dtype=np.uint64).reshape(-1, 3, len(q), orc.N)
    base = linear_part(cts3, wc, gather, q, m)
    if bias is not None:
        base[0] = W.add_mod(base[0], bias, q)
    ks = W.key_switch_reference(orc, None, keys, w, planes=digit_sums(cts3, wc, gather, q, w, m))
    return W.add_mod(base, ks, q)
