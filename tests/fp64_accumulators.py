"""Coherent worst-case sums for the FP64 accumulators of the diagonal product (k_diag_mac, k_diag_mac_resident in diag.cu) and of the
summed tensor products (k_behz_tensor_mac_fp in behz_fp.cu), and an exact model of their arithmetic.

Both kernels add fmodmul products with dadd and re-centre after every 8th term and at the end.  The sum is exact while every partial sum
stays below 2^53.  Fresh encryptions give products of random sign, whose sums grow like sqrt(L) 0.3 p, so the existing tests never come
near that limit.  The inputs here make every product of a sum the same word:

- a trivial constant ciphertext (c0 = v_l at coefficient 0 of residue l, c1 = 0) is its own rotation, word for word (the automorphism
  fixes a constant and the key switch of c1 = 0 adds zero), so every baby step and every giant step holds v_l at every NTT coefficient;
- a matrix whose kept generalised diagonals are all the weight w, with R = dim = N, has every stored diagonal equal to the constant
  plaintext w, so every lifted diagonal word is w'_l (w, or w + q_l - t above t / 2).

So each product of a group is fmodmul(v_l, w'_l), and the output is the closed form S v_l w'_l mod q_l at coefficient 0 (S the number of
(diagonal, giant step) terms), zero elsewhere and c1 = 0.  The model below evaluates fmodmul, frecenter and dadd with IEEE doubles
exactly (Python floats round every operation to nearest even; an FMA is one correctly rounded Fraction), on the kernels' sum order.

Every NTT prime p is 1 mod 2N, so (p - 1) / 2 is a multiple of N: sums of it stay exact in a double far past 2^53, and a sum that lost
its re-centre would still give the right word.  The products here are therefore odd: a double above 2^53 cannot hold an odd integer."""
import random
from fractions import Fraction

import numpy as np

TWO53 = 1 << 53
MAGIC = 6755399441055744.0  # 1.5 * 2^52, FP_MAGIC of fparith.cuh


# ---------------------------------------------------------------- fparith.cuh, operation by operation
def fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def fmodmul(a, w, p):
    """fparith.cuh fmodmul of two integer-valued doubles modulo p (pinv = 1.0 / p as the context computes it)"""
    a, w, pd = float(a), float(w), float(p)
    pinv = 1.0 / pd
    h = a * w
    lo = fma(a, w, -h)
    q = fma(h, pinv, MAGIC) - MAGIC
    return fma(-q, pd, h) + lo


def frecenter(x, p):
    pd = float(p)
    q = fma(x, 1.0 / pd, MAGIC) - MAGIC
    return fma(-q, pd, x)


def lift_weight(w, t, q):
    """the plaintext coefficient w mod t in residue q (the plain lift of multiply_plain: upper half moved up by q - t)"""
    return w + q - t if w >= (t + 1) // 2 else w


# ---------------------------------------------------------------- the kernels' sum order
def accumulate(products, period=8):
    """One accumulator of k_diag_mac / k_diag_mac_resident / k_behz_tensor_mac_fp: a = dadd(a, product) per term, a = frecenter(a) after
    every `period`-th term (None: never) and at the end.  products: (double, p) pairs or doubles with p given by the caller's closure.
    Returns (peak, value): peak the largest |a + product| an add had to hold exactly, value the kernel's final double."""
    a, peak = 0.0, 0
    for j, (r, p) in enumerate(products):
        peak = max(peak, abs(int(a) + int(r)))
        a = a + r
        if period is not None and j % period == period - 1:
            a = frecenter(a, p)
    return peak, frecenter(a, p)


def group_sum(r, p, terms, period=8):
    """(peak, word) of one accumulator that adds the same product r `terms` times; word is the canonical residue the kernel writes"""
    peak, value = accumulate([(r, p)] * terms, period)
    return peak, int(value) % p


def exact_word(r, p, terms):
    return int(r) * terms % p


# ---------------------------------------------------------------- coherent operands
def odd_half(p):
    """the product residue the coherent sums carry: (p - 3) / 2, the largest odd value below p / 2 (p = 1 mod 4)"""
    c = (p - 3) // 2
    assert c % 2 == 1
    return c


def half_operand(p, w_lift):
    """v with v w' = (p - 3) / 2 mod p"""
    return odd_half(p) * pow(w_lift, -1, p) % p


def widest_operand(p, w_lift, tries=4000, seed=0):
    """the v in [p / 2, p) among `tries` candidates whose fmodmul(v, w') has the largest magnitude and is odd: fmodmul rounds h pinv with
    an error of about (v w' / p) 2^-52, so a large v w' / p near a half-integer yields |r| beyond p / 2"""
    rng = random.Random(seed)
    best, best_r = None, 0.0
    for _ in range(tries):
        v = rng.randrange(p // 2, p)
        r = fmodmul(v, w_lift, p)
        if int(r) % 2 and abs(r) > abs(best_r):
            best, best_r = v, r
    return best


# ---------------------------------------------------------------- the diagonal product
def diag_groups(N, n1, dropped):
    """[(g, [(b, h)])] of the generalised diagonals of an R = dim = N matrix with n1 baby steps, in the stored order (g, then b, then h),
    without the (b, s) in `dropped`"""
    half = N // 2
    out = []
    for g in range(half // n1):
        keep = [(b, h) for b in (0, 1) for h in range(n1) if (b, n1 * g + h) not in dropped]
        if keep:
            out.append((g, keep))
    return out


def diag_matrix(N, w, dropped=()):
    """R = dim = N weights: w on every generalised diagonal (b, s) but the dropped ones, as floats for Engine.plain (w as a signed value)"""
    half = N // 2
    i = np.arange(N)
    b = (i[:, None] // half) ^ (i[None, :] // half)      # row (a, x), column (a ^ b, x + s)
    s = (i[None, :] % half - i[:, None] % half) % half
    M = np.full((N, N), float(w))
    for db, ds in dropped:
        M[(b == db) & (s == ds)] = 0.0
    return M


def diag_closed_form(q, v, w_lift, S, N):
    """[2][k][N] words of the product's output: c0 = S v_l w'_l mod q_l at coefficient 0, zero elsewhere, c1 = 0"""
    out = np.zeros((2, len(q), N), np.uint64)
    for l, ql in enumerate(q):
        out[0, l, 0] = S * v[l] * w_lift[l] % ql
    return out.reshape(-1)


def trivial_ct(q, c0, N, c1=None):
    """[2][k][N] words of the trivial ciphertext with constant polynomials c0 (and c1) per residue"""
    out = np.zeros((2, len(q), N), np.uint64)
    for l in range(len(q)):
        out[0, l, 0] = c0[l]
        if c1 is not None:
            out[1, l, 0] = c1[l]
    return out.reshape(-1)


def diag_model(q, v, w_lift, group_lengths, period=8):
    """per residue l: (largest peak over the groups, whether every group word equals the exact one) of the diagonal MAC's sums"""
    out = []
    for l, p in enumerate(q):
        r = fmodmul(v[l], w_lift[l], p)
        peak, ok = 0, True
        for n in set(group_lengths):
            pk, word = group_sum(r, p, n, period)
            peak, ok = max(peak, pk), ok and word == exact_word(r, p, n)
        out.append((peak, ok))
    return out


# ---------------------------------------------------------------- the summed tensor products
def tensor_operands(p):
    """(v, v2) of the columns (c0 = v, c1 = v2) and (u, u2) of the sparse elements at residue p: u = u2 = 1, so that d0 gains v = (p - 3)/2
    per term, d1 gains v + v2 = p - 4 (odd) and d2 gains v2 = (p - 5) / 2"""
    return (odd_half(p), odd_half(p) - 1), (1, 1)


def tensor_model(p, col, sp, T, period=8, lazy_reps=(0,)):
    """(peak, all words exact) of the three sums of k_behz_tensor_mac_fp over T identical terms at residue p.  lazy_reps: offsets (0 or
    -p) the forward transform's re-centring may give the lazy operands; every combination is evaluated."""
    peak, ok = 0, True
    for o in lazy_reps:
        a0, a1 = col[0] + o, col[1] + o
        b0, b1 = sp[0], sp[1]
        terms = (fmodmul(a0, b0, p), fmodmul(a0, b1, p) + fmodmul(a1, b0, p), fmodmul(a1, b1, p))
        want = ((col[0] * sp[0]), (col[0] * sp[1] + col[1] * sp[0]), (col[1] * sp[1]))
        for r, e in zip(terms, want):
            pk, word = group_sum(r, p, T, period)
            peak, ok = max(peak, pk), ok and word == e * T % p
    return peak, ok
