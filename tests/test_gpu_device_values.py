"""Values in device memory (DESIGN 4.19): cnhe_vecs_encrypt_device, cnhe_vecs_encrypt_compact_device, cnhe_vecs_decrypt_device and the
host entry points routed through them, against the Python restatement of the split and join (tests/values_ref.py).  Encryption words
are compared with cnhe_vec_from_residues of the reference split on a context seeded alike; decrypted doubles bit for bit."""
import numpy as np
import pytest

import compact_ref as cr
import values_ref as vr

pytestmark = pytest.mark.gpu

CONFIGS = {
    "n4096_p1": dict(t=[40961], N=4096, count=-1, dbc_r=10, dbc_g=20),
    "n8192_p2": dict(t=[549764251649, 549764284417], N=8192, count=-1, dbc_r=10, dbc_g=20),
    "n16384_p3_126bit": dict(t=[4398046150657, 4398044938241, 4398044577793], N=16384, count=8, dbc_r=60, dbc_g=60),
}
SEED = 515
DENSE, SPARSE = 0, 1


@pytest.fixture(scope="module", params=list(CONFIGS))
def setup(request):
    from cryptonets_b200.engine import Engine
    cfg = CONFIGS[request.param]
    eng = Engine(cfg["t"], cfg["N"], cfg["dbc_r"], cfg["dbc_g"], cfg["count"])
    eng.keygen(SEED)
    yield eng, cfg
    eng.close()


def _torch():
    return pytest.importorskip("torch")


def _edge_values(cfg, n, dim, seed):
    """random values with every edge case of the split mixed in: ties after scaling, zero, +-B/2, beyond B, negative"""
    B = vr.big_factor(cfg["t"])
    rng = np.random.default_rng(seed)
    v = rng.integers(-10 ** 6, 10 ** 6, (n, dim)).astype(np.float64) / 4  # scale 2: x.25 -> ties at .5
    wide = min(3.0 * B, 1.4e38)  # beyond B after scaling by 2, below the 1.5e38 limit
    edges = np.array([0.0, -0.0, 0.25, 0.75, -0.25, -0.75, 1.25, B / 4, -B / 4, B / 4 + 0.5, B / 2, -B / 2, wide / 2, -wide / 2, 7e37, -7e37])
    flat = v.ravel()
    pos = rng.choice(flat.size, size=min(flat.size, len(edges) * 4), replace=False)
    flat[pos] = np.resize(edges, pos.size)
    return flat.reshape(n, dim)


def _words(eng, vecs):
    return np.stack([np.stack([v.export_raw(ch, b) for ch in range(eng.P) for b in range(v.blocks)]) for v in vecs])


def _reference_vecs(eng, cfg, vals, scale):
    """the vectors of the reference split, encrypted through cnhe_vec_from_residues from seed: its residues reach the plaintexts through
    the encoder's scatter, not through the fused split-and-scatter under test"""
    eng.keygen(SEED)
    out = []
    for row in vals:
        res = np.array(vr.split(row.tolist(), scale, cfg["t"]), dtype=np.uint64)
        out.append(eng.from_residues(res, scale, DENSE, True))
    return out


def _dims(N):
    return [N // 2 + 3, N, 2 * N + 5]


def test_encrypt_words_match_reference_split(setup):
    torch = _torch()
    eng, cfg = setup
    N, scale = cfg["N"], 2.0
    for dim in _dims(N):
        vals = _edge_values(cfg, 2, dim, dim)
        ref = _words(eng, _reference_vecs(eng, cfg, vals, scale))
        eng.keygen(SEED)
        host = _words(eng, eng.encrypt_many(vals, scale))
        eng.keygen(SEED)
        dev = _words(eng, eng.encrypt_many(torch.from_numpy(vals).cuda(), scale))
        assert np.array_equal(host, ref), dim
        assert np.array_equal(dev, ref), dim


def test_single_vector_entry_points(setup):
    """cnhe_vec_encrypt, dense and sparse, against from_residues of the reference split"""
    eng, cfg = setup
    vals = _edge_values(cfg, 1, 37, 3)[0]
    for fmt in (DENSE, SPARSE):
        res = np.array(vr.split(vals.tolist(), 2.0, cfg["t"]), dtype=np.uint64)
        eng.keygen(SEED)
        ref = _words(eng, [eng.from_residues(res, 2.0, fmt, True)])
        eng.keygen(SEED)
        got = _words(eng, [eng.encrypt(vals, 2.0, fmt)])
        assert np.array_equal(got, ref), fmt


def test_compact_blob_matches_host_entry(setup):
    torch = _torch()
    eng, cfg = setup
    vals = _edge_values(cfg, 3, cfg["N"] + 9, 5)
    eng.keygen(SEED)
    host = eng.encrypt_compact(vals, 2.0)
    eng.keygen(SEED)
    dev = eng.encrypt_compact(torch.from_numpy(vals).cuda(), 2.0)
    assert dev == host
    hd = cr.parse(dev)
    assert hd is not None


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf"), 1.6e38, -1e38])
def test_out_of_range_refused_without_nonce(setup, bad):
    torch = _torch()
    from cryptonets_b200._lib import CnheError
    eng, cfg = setup
    good = _edge_values(cfg, 2, 100, 9)
    eng.keygen(SEED)
    want = _words(eng, eng.encrypt_many(good, 1.0))
    scale = 2.0 if bad == -1e38 else 1.0  # -2e38 after scaling
    eng.keygen(SEED)
    x = good.copy()
    x[1, 17] = bad
    for attempt in (lambda: eng.encrypt_many(torch.from_numpy(x).cuda(), scale), lambda: eng.encrypt_many(x, scale),
                    lambda: eng.encrypt_compact(torch.from_numpy(x).cuda(), scale)):
        with pytest.raises(CnheError) as e:
            attempt()
        assert e.value.code == -1
    assert np.array_equal(_words(eng, eng.encrypt_many(good, 1.0)), want)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _decrypt_both(eng, vecs):
    host = eng.decrypt_many(vecs)
    dev = eng.decrypt_many(vecs, device=True).cpu().numpy()
    return host, dev


def test_decrypt_every_kind_and_slabs(setup):
    eng, cfg = setup
    ts, dim = cfg["t"], 40
    rng = np.random.default_rng(21)
    rows = [rng.integers(-5000, 5000, dim) / 8.0 for _ in range(6)]
    eng.keygen(SEED)
    slab_a = eng.encrypt_many(np.stack(rows[:2]), 8.0)
    slab_b = eng.encrypt_many(np.stack(rows[2:4]), 8.0)
    vecs = [slab_b[1], slab_a[0], eng.encrypt(rows[4], 8.0, SPARSE), eng.plain(rows[5], 8.0, DENSE), eng.plain(rows[0], 8.0, SPARSE), slab_a[1]]
    order = [3, 0, 4, 5, 0, 1]
    want = np.array([vr.join(vr.split(rows[i].tolist(), 8.0, ts), 8.0, ts) for i in order])
    host, dev = _decrypt_both(eng, vecs)
    assert np.array_equal(_bits(host), _bits(want))
    assert np.array_equal(_bits(dev), _bits(want))
    for v, w in zip(vecs, want):
        assert np.array_equal(_bits(eng.decrypt(v)), _bits(w))


def test_decrypt_wide_joins_and_ties(setup):
    """residues set through from_residues whose join needs more than 53 bits, including exact ties of the conversion"""
    eng, cfg = setup
    ts = cfg["t"]
    B = vr.big_factor(ts)
    rng = np.random.default_rng(3)
    accs = [int(rng.integers(0, 2 ** 62)) * int(rng.integers(1, 2 ** 62)) % B for _ in range(61)] + [0, 1, B // 2, B // 2 + 1, B - 1]
    if B > 1 << 60:
        accs += [(1 << 54) + 2, (1 << 54) + 6, (1 << 55) + 4, B - ((1 << 54) + 2), B - ((1 << 60) + 384)]
    res = np.array([[a % t for a in accs] for t in ts], dtype=np.uint64)
    eng.keygen(SEED)
    vecs = [eng.from_residues(res, 3.0, DENSE, True), eng.from_residues(res, 3.0, SPARSE, True), eng.from_residues(res, 3.0, DENSE, False),
            eng.from_residues(res, 3.0, SPARSE, False)]
    want = np.array(vr.join(res.tolist(), 3.0, ts))
    host, dev = _decrypt_both(eng, vecs)
    for i in range(len(vecs)):
        assert np.array_equal(_bits(host[i]), _bits(want)), i
        assert np.array_equal(_bits(dev[i]), _bits(want)), i


def test_decrypt_at_a_derived_level(setup):
    eng, cfg = setup
    if eng.k < 2:
        pytest.skip("one coefficient prime: no lower level")
    vals = np.arange(-30, 30, dtype=np.float64)
    eng.keygen(SEED)
    low = eng.derive_level(eng.k - 1)
    try:
        v = eng.mod_switch(eng.encrypt_many(vals[None, :], 1.0), low)
        want = np.array(vr.join(vr.split(vals.tolist(), 1.0, cfg["t"]), 1.0, cfg["t"]))
        host, dev = _decrypt_both(low, v)
        assert np.array_equal(_bits(host[0]), _bits(want))
        assert np.array_equal(_bits(dev[0]), _bits(want))
    finally:
        low.close()


def _split(vals, scale, cfg):
    return np.array(vr.split(vals.tolist(), scale, cfg["t"]), dtype=np.uint64)


def test_decrypt_residues_every_kind(setup):
    """cnhe_vec_decrypt_residues of every kind of vector: the residues of the reference split, exactly"""
    eng, cfg = setup
    N = cfg["N"]
    eng.keygen(SEED)
    kinds = {"plain dense": (DENSE, False, N + 7), "plain sparse": (SPARSE, False, 37), "encrypted dense, one block": (DENSE, True, N // 2 + 3),
             "encrypted dense, three blocks": (DENSE, True, 2 * N + 5), "encrypted sparse": (SPARSE, True, 29)}
    for seed, (name, (fmt, enc, dim)) in enumerate(kinds.items()):
        vals = _edge_values(cfg, 1, dim, seed)[0]
        v = eng.encrypt(vals, 2.0, fmt) if enc else eng.plain(vals, 2.0, fmt)
        assert np.array_equal(eng.decrypt_residues(v), _split(vals, 2.0, cfg)), name
    if cfg["dbc_r"] <= 16:  # wider digits: the context keeps no products pending
        # a pending square: the size-3 ciphertext (c0, c1, 0) of a fresh encryption decrypts as that encryption does once relinearised
        vals = _edge_values(cfg, 1, N, 11)[0]
        fresh = eng.encrypt(vals, 2.0, DENSE)
        zero = np.zeros(eng.ct_words // 2, np.uint64)
        sq = eng.raw_import_products(np.stack([np.concatenate([fresh.export_raw(ch), zero]) for ch in range(eng.P)]), 1, N, 2.0)[0]
        assert np.array_equal(eng.decrypt_residues(sq), _split(vals, 2.0, cfg))
    if eng.k < 2:
        return
    low = eng.derive_level(eng.k - 1)
    try:
        vals = _edge_values(cfg, 1, 60, 12)[0]
        v = eng.mod_switch(eng.encrypt_many(vals[None, :], 2.0), low)[0]
        assert np.array_equal(low.decrypt_residues(v), _split(vals, 2.0, cfg))
    finally:
        low.close()


def test_force_output_in_column(setup):
    """sum_all_slots / dot_product with force_column at the first and last slot of each row: the full sum in that slot alone; column N
    is refused"""
    from cryptonets_b200._lib import CnheError
    eng, cfg = setup
    N = cfg["N"]
    rng = np.random.default_rng(12)
    a, b = rng.integers(-2, 3, N).astype(np.float64), rng.integers(-2, 3, N).astype(np.float64)
    eng.keygen(SEED)
    va, vb = eng.encrypt(a, 1.0, DENSE), eng.encrypt(b, 1.0, DENSE)
    for col in (0, N // 2 - 1, N // 2, N - 1):
        for out, total in ((eng.sum_all_slots(va, force_column=col), a.sum()), (eng.dot_product(va, vb, force_column=col), a @ b)):
            want = np.zeros(N)
            want[col] = total
            assert np.array_equal(eng.decrypt(out), want), col
    for f in (lambda: eng.sum_all_slots(va, force_column=N), lambda: eng.dot_product(va, vb, force_column=N)):
        with pytest.raises(CnheError) as e:
            f()
        assert e.value.code == -1


def test_one_wave_per_channel(setup):
    torch = _torch()
    eng, cfg = setup
    eng.keygen(SEED)
    vecs = eng.encrypt_many(np.ones((64, 50)), 1.0)
    counts = []
    for n in (1, 64):
        eng.decrypt_many(vecs[:n], device=True)
        c0 = eng.launch_count()
        eng.decrypt_many(vecs[:n], device=True)
        counts.append(eng.launch_count() - c0)
    torch.cuda.synchronize()
    assert counts[0] == counts[1]


def test_ordering_with_torch_streams(setup):
    torch = _torch()
    eng, cfg = setup
    dim = 4096
    side = torch.cuda.Stream()
    base = torch.arange(dim, dtype=torch.float64, device="cuda").repeat(3, 1)
    big = torch.randn(4096, 4096, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        for _ in range(8):
            big = big @ big / 64  # keeps the side stream busy ahead of the write below
        x = base * 2 - 7
        vecs = eng.encrypt_many(x, 1.0)
    torch.cuda.current_stream().wait_stream(side)
    out = eng.decrypt_many(vecs, device=True)
    y = out * 3  # queued at once on the current stream
    want = (np.arange(dim, dtype=np.float64) * 2 - 7) * 3
    assert np.array_equal(y.cpu().numpy(), np.tile(want, (3, 1)))


def test_refusals_key_slot_and_recording(setup):
    torch = _torch()
    from cryptonets_b200._lib import CnheError
    from cryptonets_b200.engine import Engine
    eng, cfg = setup
    eng.keygen(SEED)
    client = Engine(cfg["t"], cfg["N"], cfg["dbc_r"], cfg["dbc_g"], cfg["count"])
    try:
        client.keygen(SEED + 1)
        slot = eng.add_client_compact(client.save_compact_keys(public=False, galois=[]))
        v = eng.encrypt_many(np.ones((1, 8)), 1.0)[0]
        v.set_key_slot(slot)
        for f in (lambda: eng.decrypt_many([v]), lambda: eng.decrypt_many([v], device=True), lambda: eng.decrypt_residues(v)):
            with pytest.raises(CnheError) as e:
                f()
            assert e.value.code == -3
    finally:
        client.close()
    import ctypes as C
    from cryptonets_b200._lib import VECP, check
    from cryptonets_b200.engine import _vec_array
    x = torch.ones((2, 8), dtype=torch.float64, device="cuda")
    ok = eng.encrypt_many(np.ones((2, 8)), 1.0)
    d_out = torch.empty((2, 8), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    need = C.c_size_t()
    # the ABI calls themselves: torch may not order its streams against a stream being captured
    for f in (lambda: eng.L.cnhe_vecs_encrypt_device(eng.h, x.data_ptr(), 2, 8, 1.0, (VECP * 2)()),
              lambda: eng.L.cnhe_vecs_encrypt_compact_device(eng.h, x.data_ptr(), 2, 8, 1.0, None, 0, C.byref(need)),
              lambda: eng.L.cnhe_vecs_decrypt_device(eng.h, _vec_array(ok), 2, d_out.data_ptr(), 8)):
        eng.capture_begin()
        with pytest.raises(CnheError) as e:
            check(f())
        assert e.value.code == -3
        try:
            eng.capture_abort()
        except CnheError:
            pass
    got = eng.decrypt_many(eng.encrypt_many(x * 5, 1.0), device=True)
    assert torch.equal(got, x * 5)


def test_factory_matrices_from_tensors(setup):
    """GetEncryptedMatrix / GetEncryptedMatrixCompact of a CUDA tensor and Decrypt(device=True): the numpy path's words and values"""
    torch = _torch()
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.interfaces import EMatrixFormat
    _, cfg = setup
    f = B200BfvFactory(cfg["t"], cfg["N"], cfg["dbc_r"], cfg["dbc_g"], cfg["count"], seed=SEED)
    eng = f.engine
    m = _edge_values(cfg, 20, 7, 13)
    m[np.abs(m) > 1e6] = 1.5
    for fmt in (EMatrixFormat.ColumnMajor, EMatrixFormat.RowMajor):
        eng.keygen(SEED)
        a = f.GetEncryptedMatrix(m, fmt, 2.0)
        eng.keygen(SEED)
        b = f.GetEncryptedMatrix(torch.from_numpy(m).cuda(), fmt, 2.0)
        assert np.array_equal(_words(eng, [v.vec for v in a.vectors]), _words(eng, [v.vec for v in b.vectors]))
        dn = a.Decrypt()
        dt = b.Decrypt(device=True)
        assert dt.is_cuda and tuple(dt.shape) == dn.shape
        assert np.array_equal(_bits(dt.cpu().numpy()), _bits(dn))
        eng.keygen(SEED)
        ca = f.GetEncryptedMatrixCompact(m, fmt, 2.0)
        eng.keygen(SEED)
        assert f.GetEncryptedMatrixCompact(torch.from_numpy(m).cuda(), fmt, 2.0) == ca


def _scores(net, device):
    net.PrepareNetwork()
    return net.GetNext().Decrypt(device=True) if device else net.GetNext().Decrypt()


def test_cryptonets_end_to_end_from_a_tensor():
    """CUDA-tensor images through MatrixSource and EncryptLayer, scores decrypted into a tensor: the numpy path's scores bit for bit, and
    the Raw backend's predictions (its doubles are only good to ~2^-45 here, test_gpu_network)"""
    torch = _torch()
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import CRYPTONETS_PRIMES, cryptonets_mnist, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    imgs = synthetic_mnist(256, seed=8)
    got = {}
    for device in (False, True):
        f = B200BfvFactory(CRYPTONETS_PRIMES, 8192, seed=31)
        try:
            net, _ = cryptonets_mnist(f, torch.from_numpy(imgs).cuda() if device else imgs, timing=False)
            got[device] = _scores(net, device)
        finally:
            f.Dispose()
    assert got[True].is_cuda
    dev = got[True].cpu().numpy()
    assert np.array_equal(_bits(dev), _bits(got[False]))
    raw_net, _ = cryptonets_mnist(RawFactory(8192), imgs, timing=False)
    want = _scores(raw_net, False)
    assert np.allclose(dev, want, rtol=1e-9, atol=1e-9 * np.abs(want).max())
    assert np.array_equal(np.argmax(dev, axis=1), np.argmax(want, axis=1))


def test_lola_small_end_to_end_from_a_tensor():
    """lola_small (one more coefficient prime, where its whole network is exact) from CUDA-tensor images: the Raw backend's scores
    exactly, and the numpy path's bit for bit"""
    torch = _torch()
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import LOLA_SMALL_PRIMES, lola_small, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    imgs = synthetic_mnist(2, seed=6)
    got = {}
    for device in (False, True):
        f = B200BfvFactory(LOLA_SMALL_PRIMES, 8192, DecompositionBitCount=40, GaloisDecompositionBitCount=40, SmallModulusCount=4, seed=5)
        try:
            net, _ = lola_small(f, torch.from_numpy(imgs).cuda() if device else imgs)
            got[device] = _scores(net, device)
        finally:
            f.Dispose()
    dev = got[True].cpu().numpy()
    assert np.array_equal(_bits(dev), _bits(got[False]))
    raw_net, _ = lola_small(RawFactory(8192), imgs)
    assert np.array_equal(dev.reshape(-1), _scores(raw_net, False).reshape(-1))
