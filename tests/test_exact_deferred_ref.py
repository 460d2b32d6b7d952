"""The closed form of tests/exact_deferred_ref.py against the CPU oracle, no GPU: relinearise every size-3 product, then the scalar MAC
with a bias, word for word equal to the layer's linear part over (c0, c1) plus one key switch of the integer digit sums S_md.  This is
the identity the exact scalar-MAC path over pending squares rests on (DESIGN 4.15), here at several digit widths, with random and
maximal c2 words, both signs of weight, the centring boundary of t and padded taps."""
import numpy as np
import pytest

import exact_deferred_ref as R
import worst_case_inputs as W
from oracle.oracle_py import Oracle

CTX = {1024: (12289, W.primes(36, 1024) + W.primes(40, 1024) + W.primes(44, 1024)), 4096: (40961, None)}


@pytest.mark.parametrize("N", [1024, 4096])
@pytest.mark.parametrize("w", [4, 10, 16])
@pytest.mark.parametrize("c2", ["random", "maximal"])
def test_closed_form_equals_relinearise_then_mac(N, w, c2):
    t, q = CTX[N]
    orc = Oracle(t, N, -1, w, 20, custom_q=q)
    orc.keygen(5)
    q, k = orc.q, orc.k
    rng = np.random.default_rng(N + w + len(c2))
    n_in, M = 6, 4
    qa = np.array(q, dtype=np.uint64)[None, None, :, None]
    cts3 = (rng.integers(0, 1 << 62, (n_in, 3, k, N), dtype=np.uint64) % qa).astype(np.uint64)
    if c2 == "maximal":
        cts3[:, 2] = R.maximal_c2(q, w, N)
    else:
        cts3[0, 2] = R.maximal_c2(q, w, N)
        cts3[1, 2] = qa[0, 0] - np.uint64(1)
    relin = np.stack([orc.relinearize(cts3[j]) for j in range(n_in)])
    wres = rng.integers(0, t, (M, n_in)).astype(np.uint64)
    wres[1] = t - 1                                 # every weight -1
    wres[2, :3] = [(t + 1) // 2, (t - 1) // 2, 0]   # both sides of the centring boundary, a zero tap
    gather = np.tile(np.arange(n_in, dtype=np.int32), (M, 1))
    gather[3, ::2] = -1                             # padded taps
    bres = rng.integers(0, t, M).astype(np.uint64)
    want = orc.mac_layer(relin, gather, wres, bres, M, n_in).reshape(M, 2, k, N)
    keys = orc.relin_keys()
    wc = R.centred_weights(wres, t)
    assert wc[1].tolist() == [-1] * n_in and wc[2, :2].tolist() == [-(t - 1) // 2, (t - 1) // 2]
    for m in range(M):
        got = R.closed_form(orc, cts3, wc, gather, keys, w, m, R.bias_words(orc, np.full(N, bres[m], np.uint64)))
        assert np.array_equal(got, want[m]), m


@pytest.mark.parametrize("w", [4, 8, 9, 10, 13, 16])
def test_maximal_words_and_the_bound_edge(w):
    """maximal words: below q, every digit under the top one all ones, no larger such word; the bound edge: the largest sum of |W| with
    sum * (2^w - 1) < 2^31, so maximal digits under same-sign weights of that sum fill int32 and one more unit passes it"""
    for p in W.primes(36, 4096) + W.primes(44, 4096) + W.primes(49, 4096) + [68719403009]:
        x = R.maximal_word(p, w)
        top = (p.bit_length() - 1) // w * w
        assert x < p and x & ((1 << top) - 1) == (1 << top) - 1 and x + (1 << top) >= p
    e = R.bound_edge(w)
    assert e * ((1 << w) - 1) < 1 << 31 <= (e + 1) * ((1 << w) - 1)
    if w == 16:
        assert e == 32768 and e * 65535 == 2147450880
    ws = R.edge_weights(e)
    assert sum(ws) == e and max(ws) <= 254 and len(ws) == -(-e // 254)
