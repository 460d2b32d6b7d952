"""The FP64 path at its worst-case magnitudes (tests/worst_case_inputs.py), bit for bit against exact references:
- raw transforms on every modulus id (q, Bsk, t) of N = 4096 / 8192 / 16384, fast, SEAL-base and integer engines: forward inputs that
  push one path per output region to its analytic sum, inverse constants that double the sums up to each scheduled re-centre;
- multiply and multiply + relinearise on the BEHZ extremes (all-maximal, zero, c0-only, mont_rq words at r = 2^31 - 1, 2^31 and
  2^32 - 1), on impulses whose square is the inverse's worst constant and on forward worst cases carried into an auxiliary prime's
  residue (the square then multiplies two lazy outputs at their bound), fused and separate, both m~ conventions, among fresh
  ciphertexts in batches of 64 and with distinct operands;
- key switches with imported relinearisation keys built to make every digit's product TARGET p, on the fused path and the digit path,
  against the closed form base + INTT(sum_d NTT(digit_d) * K_d);
- the digit-decomposition corners: one digit per residue (the digit needs a reduction), 24 digits, 55 digits, and the 65-digit refusal.
tests/test_worst_case_inputs.py shows the magnitudes without the GPU.  The FP64 product stays exact well past its 2^52 operand bound
(the quotient's rounding error is absorbed by the exact remainder); what breaks first is a sum reaching 2^53.  So a dropped inverse
re-centre, which lets the sums double past 2^53 on these inputs, returns different words here, while re-centres that only keep a
product's operands below 2^52 are margin that no input can expose."""
import os

import numpy as np
import pytest

import worst_case_inputs as W

pytestmark = pytest.mark.gpu

CONFIGS = {
    "default4096": dict(t=40961, N=4096, count=-1, dbc=10),
    "cryptonets8192": dict(t=549764251649, N=8192, count=-1, dbc=10),
    "cifar16384": dict(t=957181001729, N=16384, count=8, dbc=60),
}


def _engine(name, aux="fast", dbc=None):
    from cryptonets_b200.engine import Engine
    cfg = CONFIGS[name]
    dbc = dbc or cfg["dbc"]
    saved = {v: os.environ.pop(v, None) for v in ("CNHE_AUX_BASE", "CNHE_NTT_INT")}
    if aux == "seal":
        os.environ["CNHE_AUX_BASE"] = "seal"
    if aux == "int":
        os.environ["CNHE_NTT_INT"] = "1"
    try:
        return Engine([cfg["t"]], cfg["N"], dbc, dbc, cfg["count"])
    finally:
        for v, val in saved.items():
            os.environ.pop(v, None)
            if val is not None:
                os.environ[v] = val


def _oracle(name, dbc=None):
    from oracle.oracle_py import Oracle
    cfg = CONFIGS[name]
    dbc = dbc or cfg["dbc"]
    return Oracle(cfg["t"], cfg["N"], cfg["count"], dbc, dbc)


def _mod_table(eng, orc):
    """engine modulus id -> (modulus, oracle, oracle table id)"""
    from oracle.oracle_py import Oracle
    bo = Oracle(orc.t, eng.N, custom_q=eng.bsk)
    return [(orc.q[i], orc, i) for i in range(eng.k)] + [(eng.bsk[j], bo, j) for j in range(eng.kb)] + [(orc.t, orc, 2 * orc.k + 1)]


def _worst_polys(p, o, oid, N):
    """forward worst cases for every targeted output, then the inverse constant of every scheduled segment (and p - 1)"""
    w, _, _, _, _ = o.ntt_tables(oid)
    wd = W.centred_table(w, p)
    fwd = [W.forward_worst_case(p, wd, j) for j in W.forward_path_targets(N)]
    mask = W.fp_schedule(p, N.bit_length() - 1)["inv_recenter"]
    inv = [np.full(N, W.inverse_constant(p, prev), np.uint64) for _, prev in W.inverse_segments(mask, N.bit_length() - 1)]
    return np.stack(fwd), np.stack([np.full(N, p - 1, np.uint64)] + inv)


ENGINES = [("default4096", "fast"), ("cryptonets8192", "fast"), ("cifar16384", "fast"), ("default4096", "seal"), ("cryptonets8192", "int")]


@pytest.mark.parametrize("name,aux", ENGINES, ids=["%s-%s" % e for e in ENGINES])
def test_raw_ntt_worst_case(name, aux):
    eng, orc = _engine(name, aux), _oracle(name)
    try:
        N = eng.N
        for which, (p, o, oid) in enumerate(_mod_table(eng, orc)):
            fwd, inv = _worst_polys(p, o, oid, N)
            n = len(fwd)
            d, out = eng.dev_from(fwd), eng.dev_alloc(fwd.size)
            eng.raw_ntt(d, out, n, which, 1, False)
            want = np.stack([o.ntt(oid, a) for a in fwd])
            assert np.array_equal(eng.dev_download(out, fwd.size).reshape(fwd.shape), want), (which, "forward out of place")
            eng.raw_ntt(d, d, n, which, 1, False)
            assert np.array_equal(eng.dev_download(d, fwd.size).reshape(fwd.shape), want), (which, "forward in place")
            eng.raw_ntt(out, out, n, which, 1, True)
            assert np.array_equal(eng.dev_download(out, fwd.size).reshape(fwd.shape), fwd), (which, "inverse of the forward")
            eng.dev_free(d)
            eng.dev_free(out)
            m = len(inv)
            d, out = eng.dev_from(inv), eng.dev_alloc(inv.size)
            want = np.stack([o.ntt(oid, a, inverse=True) for a in inv])
            eng.raw_ntt(d, out, m, which, 1, True)
            assert np.array_equal(eng.dev_download(out, inv.size).reshape(inv.shape), want), (which, "inverse out of place")
            eng.raw_ntt(d, d, m, which, 1, True)
            assert np.array_equal(eng.dev_download(d, inv.size).reshape(inv.shape), want), (which, "inverse in place")
            eng.dev_free(d)
            eng.dev_free(out)
    finally:
        eng.close()


def _square_impulse_ct(q, N, fresh):
    """c0 = v_l delta_0 per q residue with v_l^2 = +-TARGET q_l (its NTT is the constant v_l, its square the inverse's worst
    constant), c1 = 0; and a second one with c1 = the impulse, c0 fresh"""
    k = len(q)
    ct = np.zeros((2, k, N), np.uint64)
    ct[0, :, 0] = [W.square_root_near_target(p) for p in q]
    other = np.array(fresh, dtype=np.uint64).reshape(2, k, N).copy()
    other[1] = ct[0]
    return [ct.reshape(-1), other.reshape(-1)]


def _fresh(orc, n, seed):
    rng = np.random.default_rng(seed)
    vals = rng.integers(0, orc.t, (n, orc.N), dtype=np.uint64)
    return np.stack([orc.encrypt(orc.encode(vals[i]), 7000 + seed * 100 + i) for i in range(n)])


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("centered", [0, 1])
def test_multiply_extremes(name, centered, monkeypatch):
    from oracle.oracle_py import Oracle
    eng, orc = _engine(name), _oracle(name)
    try:
        eng.keygen(1234)
        orc.keygen(1234)
        eng.set_option("behz_centered_mtilde", centered)
        orc.set_centered_mtilde(centered)
        N, k = eng.N, eng.k
        fresh = _fresh(orc, 6, 1)
        special = W.behz_extreme_cts(orc.q, N, fresh[0]) + _square_impulse_ct(orc.q, N, fresh[1])
        bo = Oracle(orc.t, N, custom_q=eng.bsk)
        for j, out_index in ((0, N // 2 - 1), (eng.kb - 1, N // 2)):  # first auxiliary prime and m_sk
            wd_b = W.centred_table(bo.ntt_tables(j)[0], eng.bsk[j])
            special.append(W.bsk_forward_worst_ct(orc.q, eng.bsk[j], wd_b, out_index, centered))
        m = 64
        cts = np.stack([fresh[i % 6] for i in range(m)])
        where = list(range(0, m, m // len(special)))[: len(special)]
        for j, c in zip(where, special):
            cts[j] = c
        checked = sorted(set(where + [1, m - 1]))
        want3 = {i: orc.multiply(cts[i], cts[i]) for i in checked}
        want2 = {i: orc.relinearize(want3[i]) for i in checked}
        a, out3, out2 = eng.dev_from(cts), eng.dev_alloc(m * 3 * k * N), eng.dev_alloc(m * 2 * k * N)
        results = {}
        for fused in ("1", "0"):
            monkeypatch.setenv("CNHE_MUL_FUSED", fused)
            eng.raw_multiply(0, a, a, m, out3)
            got3 = eng.dev_download(out3, m * 3 * k * N).reshape(m, -1)
            eng.raw_multiply_relin(0, a, a, m, out2)
            got2 = eng.dev_download(out2, m * 2 * k * N).reshape(m, -1)
            for i in checked:
                assert np.array_equal(got3[i], want3[i]), (fused, i)
                assert np.array_equal(got2[i], want2[i]), (fused, i)
            results[fused] = (got3.copy(), got2.copy())
        assert np.array_equal(results["1"][0], results["0"][0]) and np.array_equal(results["1"][1], results["0"][1])
        # distinct operands: every extreme against the all-maximal ciphertext and against a fresh one
        b = np.stack([special[0] if i % 2 else fresh[2] for i in range(m)])
        bd = eng.dev_from(b)
        eng.raw_multiply(0, a, bd, m, out3)
        got3 = eng.dev_download(out3, m * 3 * k * N).reshape(m, -1)
        for i in checked:
            assert np.array_equal(got3[i], orc.multiply(cts[i], b[i])), ("distinct", i)
        for p in (a, bd, out3, out2):
            eng.dev_free(p)
    finally:
        eng.set_option("behz_centered_mtilde", 0)
        eng.close()


def _impulse_target_keys(q, N, dbc, all_digits):
    """(c2 residues, relinearisation keys): c2 is the impulse whose digits are all 2^dbc - 1 (the top one shorter); the keys are
    NTT-domain constants K_{d,l} with K_{d,l} * digit_d = TARGET q_l for the active digits (all of them, or digit 0 only), zero
    elsewhere, in both key parts"""
    k = len(q)
    dm = W.digit_map(q, dbc)
    c2 = np.zeros((k, N), np.uint64)
    c2[:, 0] = [(1 << (p.bit_length() - 1)) - 1 for p in q]  # every digit nonzero, all-ones below the top one
    keys = np.zeros((len(dm), 2, k, N), np.uint64)
    for d, (i, sh) in enumerate(dm):
        digit = (int(c2[i, 0]) >> sh) & ((1 << dbc) - 1)
        if (all_digits or d == 0) and digit:
            for l, p in enumerate(q):
                if digit % p:
                    keys[d, :, l, :] = W.key_constant(p, digit)
    return c2, keys


@pytest.mark.parametrize("name", ["default4096", "cryptonets8192"])
@pytest.mark.parametrize("all_digits", [False, True])
def test_key_switch_imported_keys(name, all_digits, monkeypatch):
    eng, orc = _engine(name), _oracle(name)
    try:
        eng.keygen(1234)
        orc.keygen(1234)
        N, k, q, dbc = eng.N, eng.k, orc.q, CONFIGS[name]["dbc"]
        c2, keys = _impulse_target_keys(q, N, dbc, all_digits)
        eng.import_key(0, 2, keys)
        fresh = _fresh(orc, 4, 2)
        base = np.stack([fresh[i % 4] for i in range(70)]).reshape(70, 2, k, N)
        cts3 = np.concatenate([base, np.broadcast_to(c2, (70, 1, k, N))], axis=1).reshape(70, -1).copy()
        ks = W.key_switch_reference(orc, c2, keys, dbc)
        for m in (70, 3):
            a, out = eng.dev_from(cts3[:m]), eng.dev_alloc(m * 2 * k * N)
            for fused in ("1", "0"):
                monkeypatch.setenv("CNHE_KS_FUSED", fused)
                eng.raw_relinearize(0, a, m, out)
                got = eng.dev_download(out, m * 2 * k * N).reshape(m, 2, k, N)
                for i in sorted({0, m // 2, m - 1}):
                    assert np.array_equal(got[i], W.add_mod(base[i], ks, q)), (m, fused, i)
            eng.dev_free(a)
            eng.dev_free(out)
    finally:
        eng.close()


@pytest.mark.parametrize("dbc", [37, 5, 2])
def test_decomposition_corners(dbc, monkeypatch):
    """dbc = bitlen(q_i): one digit per residue, whose mask reaches q_i (the 36-bit residues' digits need a reduction); dbc = 5: 24
    digits (a multiple of the key product's 8-digit re-centre); dbc = 2: 55 digits, near the 64-digit cap"""
    name = "default4096"
    eng, orc = _engine(name, dbc=dbc), _oracle(name, dbc=dbc)
    try:
        eng.keygen(1234)
        orc.keygen(1234)
        N, k = eng.N, eng.k
        assert eng.relin_digits == len(W.digit_map(orc.q, dbc))
        fresh = _fresh(orc, 4, 3)
        c2 = W.digit_worst_case_target(orc.q, dbc, lambda l: W.centred_table(orc.ntt_tables(l)[0], orc.q[l]), N - 1)
        m = 64
        cts3 = np.stack([orc.multiply(fresh[i % 4], fresh[(i + 1) % 4]) for i in range(4)])
        cts3 = np.stack([cts3[i % 4] for i in range(m)]).reshape(m, 3, k, N)
        cts3[0, 2] = c2
        cts3[m - 1, 2] = np.array(orc.q, dtype=np.uint64)[:, None] - np.uint64(1)
        cts3 = cts3.reshape(m, -1)
        want = {i: orc.relinearize(cts3[i]) for i in (0, 1, m - 1)}
        a, out = eng.dev_from(cts3), eng.dev_alloc(m * 2 * k * N)
        results = {}
        for fused in ("1", "0"):
            monkeypatch.setenv("CNHE_KS_FUSED", fused)
            eng.raw_relinearize(0, a, m, out)
            got = eng.dev_download(out, m * 2 * k * N).reshape(m, -1)
            for i, w in want.items():
                assert np.array_equal(got[i], w), (fused, i)
            results[fused] = got.copy()
        assert np.array_equal(results["1"], results["0"])
        eng.dev_free(a)
        eng.dev_free(out)
    finally:
        eng.close()


def test_too_many_digits_is_refused():
    import torch
    from cryptonets_b200._lib import CnheError
    torch.cuda.init()
    free0, _ = torch.cuda.mem_get_info()
    for _ in range(3):
        with pytest.raises(CnheError, match="more than 64 digits"):
            _engine("default4096", dbc=1)
    free1, _ = torch.cuda.mem_get_info()
    assert free0 - free1 < 64 << 20, "refused contexts left device memory behind"
    eng = _engine("default4096")
    eng.keygen(1)
    eng.close()
