"""Reference BFV modulus switch (SEAL's Evaluator::mod_switch_scale_to_next), in Python integers: the checker of cnhe_vecs_mod_switch.

mod_switch drops the last prime of a residue array one step at a time exactly as the CUDA kernel does, on the residues only;
mod_switch_big computes the same words from the big integer x in [0, q) of every coefficient, as floor((x + floor(q_j / 2)) / q_j) per
dropped prime.  The two share no code, so their agreement checks the residue formula itself."""
from functools import reduce

import numpy as np


def mod_switch(words, q, k_out):
    """words [..., k, N] (canonical residues mod q[0..k-1]) -> [..., k_out, N]: primes q[k-1] .. q[k_out] dropped in turn."""
    a = np.asarray(words, dtype=np.uint64)
    k = len(q)
    assert a.shape[-2] == k and 1 <= k_out <= k
    x = [a[..., l, :].astype(object) for l in range(k)]
    for j in range(k - 1, k_out - 1, -1):
        half = q[j] >> 1
        r = (x[j] + half) % q[j]
        for i in range(j):
            x[i] = ((x[i] - r % q[i] + half % q[i]) * pow(q[j], -1, q[i])) % q[i]
    return np.stack([np.asarray(x[l], dtype=np.uint64) for l in range(k_out)], axis=-2)


def compose(words, q):
    """[k, N] residues -> list of N integers in [0, prod q) (CRT)."""
    Q = reduce(lambda u, v: u * v, q)
    out = [0] * words.shape[-1]
    for l, p in enumerate(q):
        c = (Q // p) * pow((Q // p) % p, -1, p)
        for n, v in enumerate(words[l]):
            out[n] = (out[n] + int(v) * c) % Q
    return out


def mod_switch_big(poly, q, k_out):
    """One polynomial [k, N] switched on big integers: x -> floor((x + floor(q_j / 2)) / q_j) for j = k-1 .. k_out, then reduced."""
    xs = compose(np.asarray(poly, dtype=np.uint64), q)
    for j in range(len(q) - 1, k_out - 1, -1):
        xs = [(x + (q[j] >> 1)) // q[j] for x in xs]
    return np.array([[x % q[l] for x in xs] for l in range(k_out)], dtype=np.uint64)
