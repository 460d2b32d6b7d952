"""The scalar-MAC layer at its accumulator bounds: each kernel at the largest layer its gate admits, and the next kernel just past it.

mac_channel (csrc/vec.cu) serves each plaintext channel with wgmma, mma.sync, FP64 or the 128-bit integer MAC, whichever is first to
hold its bound (tests/mac_bounds.py restates the gates).  Every case here:
  - asserts the kernel that served each channel from the `[mac route ...]` line CNHE_MAC_ROUTE prints, so a silent fallback cannot pass;
  - checks every output word against the closed form of tests/mac_bounds.py, and against the CPU oracle where the layer is small;
  - reruns the layer with the faster kernels switched off (CNHE_MAC_NO_UMMA, CNHE_MAC_NO_IMMA, CNHE_MAC_INT) and requires the same words;
  - feeds coherent worst cases: every tap reads a word that is maximal for the kernel's cut (255 in every limb but the top one, 2^26 - 1
    in the FP64 low half, q - 1 for the integer MAC), each row's weights share one sign, and rows alternate between all-positive and
    all-negative, so the sums reach both ends of the int32 or 2^52 range; biases are negative constants.
The large-K layers read one to three inputs over and over, so they stay in L2 and take milliseconds."""
import re

import numpy as np
import pytest

import mac_bounds as B
from cryptonets_b200._lib import CnheError
from cryptonets_b200.engine import DENSE, SPARSE, Engine

pytestmark = pytest.mark.gpu

ERR_INVALID = -1
N = 4096
T = 786433  # = 1 mod 2^18: a weight of 131071 or 131072 is itself, not its negative
KERNEL_ENV = ("CNHE_MAC_NO_UMMA", "CNHE_MAC_NO_IMMA", "CNHE_MAC_INT", "CNHE_MAC_ROUTE", "CNHE_UMMA_PROF")
ROUTE = re.compile(r"\[mac route ch=(\d+) kernel=(\w+) K=(\d+) M=(\d+)\]")
# the kernel each switch leaves for a layer that `route` would give to `kernel`
FALLBACK = {"CNHE_MAC_NO_UMMA": {"umma": "imma"}, "CNHE_MAC_NO_IMMA": {"umma": "fp64", "imma": "fp64"},
            "CNHE_MAC_INT": {"umma": "int128", "imma": "int128", "fp64": "int128"}}


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    for v in KERNEL_ENV:
        monkeypatch.delenv(v, raising=False)


_ENGINES = {}


@pytest.fixture(scope="module")
def ctx():
    """ctx(bits, t=(T,)): a context on two `bits`-bit primes at N = 4096, one per parameter set for the whole module"""
    def get(bits, t=(T,)):
        key = (bits, tuple(t))
        if key not in _ENGINES:
            eng = Engine(list(t), N, 10, 20, -1, coeff_moduli=B.primes(bits, N, 2))
            eng.keygen(29)
            _ENGINES[key] = eng
        return _ENGINES[key]
    yield get
    for eng in _ENGINES.values():
        eng.close()
    _ENGINES.clear()


def _words(eng, n, kind, seed):
    """[n][2][k][N] words, the same in every channel.  kind "limb": 0xff in every byte below the top limb, "half": the FP64 low half at
    2^26 - 1, "top": q - 1.  Coefficients 1 mod 3 of "limb" and "half" words take a random top part, so the output is not one word."""
    rng = np.random.default_rng(seed)
    maxbits = max(p.bit_length() for p in eng.q)
    out = np.zeros((n, 2, eng.k, N), dtype=np.uint64)
    for l, p in enumerate(eng.q):
        if kind == "top":
            out[:, :, l] = p - 1
            continue
        s = 8 * (B.limbs(maxbits) - 1) if kind == "limb" else B.FP64_SPLIT
        out[:, :, l] = B.maximal_limb_word(p, maxbits) if kind == "limb" else B.maximal_low_half_word(p)
        rnd = rng.integers(0, p >> s, (n, 2, len(range(1, N, 3))), dtype=np.uint64)
        out[:, :, l, 1::3] = (rnd << np.uint64(s)) | np.uint64((1 << s) - 1)
    return out


def _import(eng, words, slab=True):
    """one allocation of evenly spaced rows (slab), or one allocation per input, made in a scrambled order so that the inputs are never
    evenly spaced rows"""
    n = words.shape[0]
    per_ch = np.broadcast_to(words, (eng.P,) + words.shape)
    if slab:
        return eng.import_raw_many(np.ascontiguousarray(per_ch), n, 1, N, 1.0)
    ins = {}
    for i in np.random.default_rng(n).permutation(n) if n > 2 else range(n):
        ins[i] = eng.import_raw(np.ascontiguousarray(per_ch[:, i]), 1, N, 1.0)
    return [ins[i] for i in range(n)]


def _signed_rows(M, K, mag):
    """all-positive even rows, all-negative odd rows, of magnitude mag"""
    return np.where(np.arange(M)[:, None] % 2 == 0, mag, -mag) * np.ones((M, K), dtype=np.int64)


def _bias(M):
    return -np.array([T // 2 - m for m in range(M)], dtype=np.int64)  # negative, the largest magnitude first


def _run(eng, capfd, monkeypatch, ins, gather, w, bias, env=None, act=False):
    """the layer's outputs [M][P][2kN] and the kernel of every channel"""
    M, K = gather.shape
    wv = [eng.plain(w[m].astype(np.float64), 1.0, SPARSE) for m in range(M)]
    bv = None if bias is None else [eng.plain(np.full(N, float(bias[m])), 1.0, DENSE) for m in range(M)]
    monkeypatch.setenv("CNHE_MAC_ROUTE", "1")
    if env:
        monkeypatch.setenv(env, "1")
    capfd.readouterr()
    try:
        if act:
            outs = eng.layer_activation_conv_dense(ins, None, None, None, gather, wv, bv, M, K)
        else:
            outs = eng.layer_conv_dense(ins, gather, wv, bv, M, K)
        eng.sync()
    finally:
        monkeypatch.delenv("CNHE_MAC_ROUTE")
        if env:
            monkeypatch.delenv(env)
        eng.dispose_many(wv + (bv or []))
    lines = ROUTE.findall(capfd.readouterr().err)
    assert [int(x[0]) for x in lines] == list(range(eng.P)), lines
    assert all((int(x[2]), int(x[3])) == (K, M) for x in lines), lines
    words = np.stack([np.stack([o.export_raw(ch, 0) for ch in range(eng.P)]) for o in outs])
    eng.dispose_many(outs)
    return words, [x[1] for x in lines]


def _check(eng, capfd, monkeypatch, ins, words, gather, w, bias, routes, oracle=False, w_ch=None, act=False):
    """run the layer, assert its routes, its words against the closed form (and the oracle), and the same words with each faster kernel
    switched off; w_ch: per-channel signed weights when they differ from w"""
    M = gather.shape[0]
    got, seen = _run(eng, capfd, monkeypatch, ins, gather, w, bias, act=act)
    assert seen == routes, (seen, routes)
    for ch in range(eng.P):
        wc = w if w_ch is None else w_ch[ch]
        t = eng.primes[ch]
        want = B.mac_closed_form(words, gather, wc, None if bias is None else B.centred(bias, t), eng.q, t).reshape(M, -1)
        assert np.array_equal(got[:, ch], want), ch
        if oracle:
            from oracle.oracle_py import Oracle
            orc = Oracle(t, N, custom_q=eng.q)
            wo = orc.mac_layer(words.reshape(words.shape[0], -1), gather, B.residues(B.centred(wc, t), t),
                               None if bias is None else B.residues(B.centred(bias, t), t), M, gather.shape[1], threads=8).reshape(M, -1)
            assert np.array_equal(got[:, ch], wo), ch
    for env, fall in FALLBACK.items():
        again, seen2 = _run(eng, capfd, monkeypatch, ins, gather, w, bias, env=env, act=act)
        assert seen2 == [fall.get(r, r) for r in routes], (env, seen2)
        assert np.array_equal(again, got), env
    return got


# ---------------------------------------------------------------- mma.sync at its int32 gate
@pytest.mark.parametrize("bits", [40, 48, 50])
def test_imma_at_its_int32_gate(ctx, capfd, monkeypatch, bits):
    """K = 33155 taps of weight +-254 over one to three maximal-limb inputs: W1 = W2 = 127 per tap, both into one int32 accumulator, so
    every limb sum below the top one reaches 33155 * 254 * 255 = 2,147,449,350 against 2^31 - 1.  K = 33156 goes to FP64, same words.
    5, 6 and 7 limbs (40-, 48- and 50-bit primes) instantiate the kernel's three bodies."""
    eng = ctx(bits)
    n = {40: 1, 48: 2, 50: 3}[bits]
    words = _words(eng, n, "limb", bits)
    ins = _import(eng, words, slab=False)
    M = 24  # two m16 tiles, the second half full
    for K, kernel in ((B.largest(B.imma_admits, 32), "imma"), (B.largest(B.imma_admits, 32) + 1, "fp64")):
        assert B.route(K, M, bits, 254) == kernel
        gather = np.tile(np.arange(K, dtype=np.int32) % n, (M, 1))
        _check(eng, capfd, monkeypatch, ins, words, gather, _signed_rows(M, K, 254), _bias(M), [kernel])
    eng.dispose_many(ins)


def test_imma_gate_on_size_three_products(ctx, capfd, monkeypatch):
    """the square followed by the layer (cnhe_layer_activation_conv_dense): mma.sync sums the size-3 products c0, c1 and the reduced c2
    at K = 33155; the outputs are the relinearised closed form over the oracle's products, word for word"""
    from oracle.oracle_py import Oracle
    eng = ctx(50)
    orc = Oracle(T, N, -1, 10, 20, custom_q=eng.q)
    orc.keygen(29)
    rng = np.random.default_rng(5)
    n, M, K = 2, 8, B.largest(B.imma_admits, 32)
    vals = rng.integers(0, T, (n, N), dtype=np.uint64)
    cts = np.stack([orc.encrypt(orc.encode(vals[i]), 300 + i) for i in range(n)])
    ins = [eng.import_raw(cts[i], 1, N, 1.0) for i in range(n)]
    prods = np.stack([orc.multiply(cts[i], cts[i]) for i in range(n)]).reshape(n, 3, eng.k, N)
    gather = np.tile(np.arange(K, dtype=np.int32) % n, (M, 1))
    w, bias = _signed_rows(M, K, 254), _bias(M)
    y3 = B.mac_closed_form(prods, gather, w, bias, eng.q, T)
    want = np.stack([orc.relinearize(y3[m].reshape(-1)) for m in range(M)])
    got, seen = _run(eng, capfd, monkeypatch, ins, gather, w, bias, act=True)
    assert seen == ["imma"]
    assert np.array_equal(got[:, 0], want)
    for env in FALLBACK:
        again, _ = _run(eng, capfd, monkeypatch, ins, gather, w, bias, env=env, act=True)
        assert np.array_equal(again, got), env
    eng.dispose_many(ins)


# ---------------------------------------------------------------- FP64 at its 2^52 gate
def test_fp64_at_its_2_52_gate(ctx, capfd, monkeypatch):
    """|w| = 131071 over words whose low 26 bits are all ones: K = 512 puts each low-half sum at 512 * 131071 * (2^26 - 1), just under 2^52,
    on the FP64 kernel; K = 513, and K = 512 at |w| = 131072, go to the 128-bit MAC.  K = 2047 (sums near 2^54, beyond a double's 53 bits)
    must stay there too.  Same words everywhere."""
    eng = ctx(50)
    words = _words(eng, 2, "half", 1)
    ins = _import(eng, words, slab=False)
    M = 8
    for K, mag, kernel, oracle in ((512, 131071, "fp64", True), (513, 131071, "int128", False), (512, 131072, "int128", False),
                                   (2047, 131071, "int128", False)):
        assert B.route(K, M, 50, mag) == kernel
        gather = np.tile(np.arange(K, dtype=np.int32) % 2, (M, 1))
        _check(eng, capfd, monkeypatch, ins, words, gather, _signed_rows(M, K, mag), _bias(M), [kernel], oracle=oracle)
    eng.dispose_many(ins)


# ---------------------------------------------------------------- wgmma at its shared-memory edge
@pytest.mark.parametrize("bits", [40, 48, 50])
def test_wgmma_at_its_shared_memory_edge(ctx, capfd, monkeypatch, bits):
    """the widest all-+-254 dense window the planner fits (every tap also in the W2 scratch slab) on a slab of maximal-limb words, then one
    chunk more, which has no plan and goes to mma.sync.  Each limb count instantiates its own epilogue."""
    eng = ctx(bits)
    limbs = B.limbs(bits)
    Kw = B.widest_umma_window(limbs)
    words = _words(eng, Kw + 32, "limb", bits + 1)
    ins = _import(eng, words)
    M = 16
    for K, kernel in ((Kw, "umma"), (Kw + 32, "imma")):
        gather, w = B.wide_dense(M, K)
        assert (B.umma_plan(gather, w, limbs) is not None) == (kernel == "umma")
        _check(eng, capfd, monkeypatch, ins, words, gather, w, _bias(M), [kernel], oracle=bits == 48)
    eng.dispose_many(ins)


def test_duplicate_taps_under_wgmma(ctx, capfd, monkeypatch):
    """the planner merges taps that read one input: +200 and -100 merge to 100 and stay on wgmma; +200 and +100 merge to 300, past the
    +-254 a weight byte pair holds, so the layer leaves wgmma (for mma.sync, which takes each tap on its own)"""
    eng = ctx(40)
    n_in, M = 40, 8
    words = _words(eng, n_in, "limb", 7)
    ins = _import(eng, words)
    K = 2 * n_in
    gather = np.tile(np.repeat(np.arange(n_in, dtype=np.int32), 2), (M, 1))  # every input twice
    for second, kernel in ((-100, "umma"), (100, "imma")):
        w = np.tile(np.array([200, second] * n_in), (M, 1)) * np.where(np.arange(M)[:, None] % 2 == 0, 1, -1)
        _check(eng, capfd, monkeypatch, ins, words, gather, w, _bias(M), [kernel], oracle=True)
    eng.dispose_many(ins)


# ---------------------------------------------------------------- each term of the tensor-core predicates, once
@pytest.mark.parametrize("edge", ["maxbits-32-33", "maxbits-50-51", "M-7-8", "K-31-32"])
def test_predicate_edges(ctx, capfd, monkeypatch, edge):
    """dense layers over separate inputs (no slab, so mma.sync or below): 4 -> 5 limbs, 50 -> 51 bits, 7 -> 8 outputs, 31 -> 32 taps"""
    rng = np.random.default_rng(11)
    cases = {"maxbits-32-33": [(32, 8, 32, "fp64"), (33, 8, 32, "imma")], "maxbits-50-51": [(50, 8, 32, "imma"), (51, 8, 32, "int128")],
             "M-7-8": [(40, 7, 32, "fp64"), (40, 8, 32, "imma")], "K-31-32": [(40, 8, 31, "fp64"), (40, 8, 32, "imma")]}[edge]
    for bits, M, K, kernel in cases:
        assert B.route(K, M, bits, 254) == kernel
        eng = ctx(bits)
        words = _words(eng, K, "limb" if bits > 32 else "top", bits)
        ins = _import(eng, words, slab=False)
        gather = np.tile(rng.permutation(K).astype(np.int32), (M, 1))
        w = _signed_rows(M, K, 1) * rng.integers(1, 255, (M, K))
        w[0, :], w[1, :] = 254, -254
        _check(eng, capfd, monkeypatch, ins, words, gather, w, _bias(M), [kernel], oracle=True)
        eng.dispose_many(ins)


def test_slab_with_one_row_out_of_place(ctx, capfd, monkeypatch):
    """wgmma reads its inputs as evenly spaced rows of one slab: the same layer with two rows swapped in the input list is not a slab and
    goes to mma.sync, with the same words for the same taps"""
    eng = ctx(40)
    n_in, M = 64, 8
    words = _words(eng, n_in, "limb", 3)
    ins = _import(eng, words)
    gather = np.tile(np.arange(n_in, dtype=np.int32), (M, 1))
    w = _signed_rows(M, n_in, 254)
    _check(eng, capfd, monkeypatch, ins, words, gather, w, _bias(M), ["umma"])
    order = np.arange(n_in)
    order[[5, 6]] = order[[6, 5]]
    _check(eng, capfd, monkeypatch, [ins[i] for i in order], words[order], gather, w, _bias(M), ["imma"])
    eng.dispose_many(ins)


# ---------------------------------------------------------------- the 128-bit MAC at its refusal
@pytest.mark.parametrize("bits", [56, 60])
def test_int128_at_its_refusal(ctx, capfd, monkeypatch, bits):
    """words q - 1 and weights -1 (and +1 on the other rows): each product is (q - 1)^2, and 2 maxbits + bits(K) <= 127 admits K = 32767 at
    56 bits and 127 at 60 bits.  The next K is refused with CNHE_ERR_INVALID and the context keeps working."""
    eng = ctx(bits)
    K = B.largest(lambda k: B.int128_admits(k, bits))
    n = 3 if bits == 56 else 2
    words = _words(eng, n, "top", 0)
    ins = _import(eng, words, slab=False)
    M = 8
    w = -_signed_rows(M, K, 1)
    gather = np.tile(np.arange(K, dtype=np.int32) % n, (M, 1))
    assert B.route(K, M, bits, 1) == "int128"
    got = _check(eng, capfd, monkeypatch, ins, words, gather, w, _bias(M), ["int128"], oracle=bits == 60)
    wv = [eng.plain(np.full(K + 1, -1.0), 1.0, SPARSE) for _ in range(M)]
    with pytest.raises(CnheError) as e:
        eng.layer_conv_dense(ins, np.tile(np.arange(K + 1, dtype=np.int32) % n, (M, 1)), wv, None, M, K + 1)
    assert e.value.code == ERR_INVALID and "128-bit" in str(e.value)
    eng.dispose_many(wv)
    again, seen = _run(eng, capfd, monkeypatch, ins, gather, w, _bias(M))
    assert seen == ["int128"] and np.array_equal(again, got)
    eng.dispose_many(ins)


# ---------------------------------------------------------------- one call, two kernels
def test_routing_per_channel(ctx, capfd, monkeypatch):
    """two plaintext primes: every weight is 65537 + s (|s| <= 127), which is s modulo 65537 (wgmma) and itself modulo 786433 (FP64).
    One call routes the channels apart, and each matches the closed form of its own weights"""
    t2 = 65537
    eng = ctx(40, t=(T, t2))
    rng = np.random.default_rng(13)
    n_in, M = 64, 8
    words = _words(eng, n_in, "limb", 13)
    ins = _import(eng, words)
    gather = np.tile(np.arange(n_in, dtype=np.int32), (M, 1))
    w = _signed_rows(M, n_in, 1) * (t2 + rng.integers(1, 128, (M, n_in)))
    w_ch = [B.centred(w, t) for t in (T, t2)]
    assert np.abs(w_ch[0]).max() > 254 and np.abs(w_ch[1]).max() <= 127
    _check(eng, capfd, monkeypatch, ins, words, gather, w, _bias(M), ["fp64", "umma"], oracle=True, w_ch=w_ch)
    eng.dispose_many(ins)
