"""The single-vector rotate, duplicate and permute calls word for word against the CPU oracle's composition of the same operations, and their
operation counts against that composition's.  Each single call is its batched form (cnhe_vecs_rotate, cnhe_vecs_duplicate_batch,
cnhe_vecs_permute_batch) with one vector, so the oracle is their independent reference."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PRIMES, N = [2277377, 2424833], 8192  # LoLa-small's plaintext primes: two channels
P = len(PRIMES)
SEED, CLIENT_SEED = 310, 420


def _oracles(seed):
    """One oracle per channel, keyed as the engine keys that channel (seed + channel)."""
    from oracle.oracle_py import Oracle
    orcs = []
    for ch, t in enumerate(PRIMES):
        o = Oracle(t, N, -1, 10, 20)
        o.keygen(seed + ch)
        orcs.append(o)
    return orcs


@pytest.fixture(scope="module")
def ctx():
    from cryptonets_b200.engine import Engine
    eng = Engine(PRIMES, N, 10, 20, -1)
    eng.keygen(SEED)
    orcs = _oracles(SEED)
    assert orcs[0].q == eng.q
    yield eng, orcs
    eng.close()


def _naf(value):
    """non-adjacent form of a rotation amount (SEAL util::naf), as tests/test_gpu_network.py counts hops"""
    v, i = abs(value), 0
    while v:
        z = (2 - (v & 3)) if (v & 1) else 0
        v = (v - z) >> 1
        if z:
            yield z * (1 << i)
        i += 1


def _hops(orc, elts, steps):
    """Key switches of a row rotation: none for 0, one when the step has its own key, else one per NAF term except a half-row one"""
    if steps == 0:
        return 0
    if orc.galois_elt_from_step(steps) in elts:
        return 1
    return sum(1 for h in _naf(steps) if abs(h) != N // 2)


def _counted(eng, fn):
    """fn()'s result and the operations it counted"""
    eng.op_counts(reset=True)
    out = fn()
    return out, eng.op_counts(reset=True)


def _ops(rot=0, col=0, plain=0, add=0):
    return dict(Rotation=P * rot, ColumnRotation=P * col, PlainMultiplication=P * plain, Addition=P * add)


def _only(counts, want):
    """the counts equal want's and nothing else was counted"""
    return {k: v for k, v in counts.items() if v} == {k: v for k, v in want.items() if v}


# ------------------------------------------------------------------------------------------------ rotate
AMOUNTS = [0, 1, -1, 3, 5, -1024]  # 3 and 5: NAF hops, their elements have no key of their own


@pytest.mark.parametrize("amount", AMOUNTS)
def test_rotate_equals_the_oracle(ctx, amount):
    eng, orcs = ctx
    x = eng.encrypt(np.random.default_rng(amount % 97).integers(0, 1000, N // 2).astype(np.float64))
    y, counts = _counted(eng, lambda: eng.rotate(x, amount))
    assert (y.dim, y.scale, y.blocks, y.key_slot) == (N // 2, 1.0, 1, 0)
    for ch, orc in enumerate(orcs):
        assert np.array_equal(y.export_raw(ch, 0), orc.rotate_rows(x.export_raw(ch, 0), amount)), ch
    elts = set(eng.galois_elts())
    assert _only(counts, _ops(rot=_hops(orcs[0], elts, amount))), counts
    eng.dispose_many([x, y])


def test_rotate_on_a_client_slot_equals_the_oracle(ctx):
    """A client's key slot holds the Galois keys of its compact blob, fresh pairs over its secret key: the oracle keyed with the client's
    seed takes those keys (read from a context loaded from the same blob) and rotates with them."""
    from cryptonets_b200.engine import Engine
    eng, server_orcs = ctx
    elts = sorted({server_orcs[0].galois_elt_from_step(s) for s in (1, -1, 4, -1024)})  # every hop of AMOUNTS
    client = Engine(PRIMES, N, 10, 20, -1)
    client.keygen(CLIENT_SEED)
    blob = client.save_compact_keys(public=False, galois=elts)
    client.close()
    orcs = _oracles(CLIENT_SEED)
    held = Engine(None, compact_keys=blob)
    try:
        for ch, orc in enumerate(orcs):
            for e in elts:
                orc.set_galois_key(e, held.export_key(ch, 3, e))
    finally:
        held.close()
    slot = eng.add_client_compact(blob)
    try:
        x = eng.encrypt(np.random.default_rng(9).integers(0, 1000, N // 2).astype(np.float64))
        xc = eng.copy(x)
        xc.set_key_slot(slot)
        for amount in AMOUNTS:
            y, counts = _counted(eng, lambda: eng.rotate(xc, amount))
            assert y.key_slot == slot
            for ch, orc in enumerate(orcs):
                want = orc.rotate_rows(x.export_raw(ch, 0), amount)
                assert np.array_equal(y.export_raw(ch, 0), want), (amount, ch)
                if amount:
                    assert not np.array_equal(want, server_orcs[ch].rotate_rows(x.export_raw(ch, 0), amount)), (amount, ch)
            assert _only(counts, _ops(rot=_hops(orcs[0], set(elts), amount))), (amount, counts)
            y.dispose()
        eng.dispose_many([x, xc])
    finally:
        eng.remove_client(slot)


# ------------------------------------------------------------------------------------------------ duplicate
@pytest.mark.parametrize("dim,count", [(1000, 8), (300, 4), (4096, 2)])
def test_duplicate_equals_the_oracle(ctx, dim, count):
    """Duplicate (AtomicSealBfvVector.cs:1370-1408): the copies whose offset reaches the second row rotate the column-rotated input back by
    half a row; 1024 x 8 and 4096 x 2 take the column rotation, 512 x 4 does not."""
    eng, orcs = ctx
    x = eng.encrypt(np.random.default_rng(dim).integers(0, 1000, dim).astype(np.float64))
    y, counts = _counted(eng, lambda: eng.duplicate(x, count))
    shift = 1 << (dim - 1).bit_length()
    assert (y.dim, y.scale, y.blocks, y.key_slot) == (count * shift, 1.0, 1, 0)
    steps = []
    for i in range(1, count):
        target = i * shift
        steps.append((target * 2 >= N, -(target - N // 2 if target * 2 >= N else target)))
    column = any(c for c, _ in steps)
    for ch, orc in enumerate(orcs):
        ct = x.export_raw(ch, 0)
        rotator = orc.rotate_columns(ct) if column else None
        want = ct
        for c, s in steps:
            want = orc.add(want, orc.rotate_rows(rotator if c else ct, s))
        assert np.array_equal(y.export_raw(ch, 0), want), ch
    elts = set(eng.galois_elts())
    assert _only(counts, _ops(rot=sum(_hops(orcs[0], elts, s) for _, s in steps), col=int(column), add=count - 1)), counts
    eng.dispose_many([x, y])


# ------------------------------------------------------------------------------------------------ permute
def _permute_case(eng, seed):
    """An input, and one permutation with a NULL selection, negative shifts and one selection vector used twice"""
    rng = np.random.default_rng(seed)
    x = eng.encrypt(rng.integers(0, 1000, N // 2).astype(np.float64))
    masks = [(rng.random(N // 2) < 0.3).astype(np.float64) for _ in range(3)]
    plains = [eng.plain(m) for m in masks]
    sel = [plains[0], None, plains[1], plains[0], plains[2]]
    shifts = [3, 0, -17, -1024, 5]
    mask_of = [masks[0], None, masks[1], masks[0], masks[2]]
    return x, plains, sel, shifts, mask_of


def test_permute_equals_the_oracle(ctx):
    """Permute (AtomicSealBfvVector.cs:1436-1475): multiply_plain, rotate_rows(shift), add for every non-NULL selection in order."""
    eng, orcs = ctx
    x, plains, sel, shifts, mask_of = _permute_case(eng, 5)
    y, counts = _counted(eng, lambda: eng.permute(x, sel, shifts, 2000))
    assert (y.dim, y.scale, y.blocks, y.key_slot) == (2000, 1.0, 1, 0)
    for ch, orc in enumerate(orcs):
        ct = x.export_raw(ch, 0)
        want = None
        for m, s in zip(mask_of, shifts):
            if m is None:
                continue
            r = orc.rotate_rows(orc.multiply_plain(ct, orc.encode(m.astype(np.uint64))), s)
            want = r if want is None else orc.add(want, r)
        assert np.array_equal(y.export_raw(ch, 0), want), ch
    terms = [s for m, s in zip(mask_of, shifts) if m is not None]
    elts = set(eng.galois_elts())
    assert _only(counts, _ops(rot=sum(_hops(orcs[0], elts, s) for s in terms), plain=len(terms), add=len(terms) - 1)), counts
    eng.dispose_many([x, y] + plains)


def test_batched_permute_counts_every_term(ctx):
    """One PlainMultiplication per (client, permutation, non-NULL selection), a selection listed twice included, as B single calls count."""
    eng, orcs = ctx
    x, plains, sel, shifts, mask_of = _permute_case(eng, 6)
    x2 = eng.copy(x)
    ys, counts = _counted(eng, lambda: eng.permute_many([x, x2], [(sel, shifts)] * 2, 2000))
    terms = sum(m is not None for m in mask_of)
    assert counts["PlainMultiplication"] == P * 2 * 2 * terms, counts
    eng.dispose_many(ys + [x, x2] + plains)
