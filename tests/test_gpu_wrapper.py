"""The reference's own known-answer tests, restated on the GPU backend: `HE Wrapper Tests/BasicOperations.cs` (default factory:
N=4096, primes {40961,65537,114689,147457,188417}, IFactory.cs:247-253) and the BasicExample of README.md:61-73.
Decrypted results must equal the plain results exactly, as in the reference (`Compare`, BasicOperations.cs:41-55)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

values1 = np.array([-1, 9, 3, 20, 1000, -6945], dtype=np.float64)
values2 = np.array([8, -22, 5, 4, 254, -12], dtype=np.float64)
values_m = np.array([[1, -2, 3, -44, 5, 7], [99, 12, -88, 22, 16, 13]], dtype=np.float64)
scale = 12


@pytest.fixture(scope="module")
def F():
    from cryptonets_b200.he import B200BfvFactory
    f = B200BfvFactory()
    yield f
    f.Dispose()


@pytest.fixture(scope="module")
def objs(F):
    from cryptonets_b200.interfaces import EMatrixFormat, EVectorFormat
    return dict(enc1=F.GetEncryptedVector(values1, EVectorFormat.dense, scale), enc2=F.GetEncryptedVector(values2, EVectorFormat.dense, scale),
                plain2=F.GetPlainVector(values2, EVectorFormat.dense, scale), mat=F.GetEncryptedMatrix(values_m, EMatrixFormat.ColumnMajor, scale))


def test_decrypt(F, objs):
    assert np.array_equal(objs["enc1"].Decrypt(), values1)
    assert np.array_equal(objs["mat"].Decrypt(), values_m)
    assert np.array_equal(objs["mat"].GetColumn(0).Decrypt(), values_m[:, 0])


def test_matrix_vector_multiplication(F, objs):
    from cryptonets_b200.interfaces import EVectorFormat
    enc_sparse = F.GetEncryptedVector(values1, EVectorFormat.sparse, scale)
    assert np.array_equal(objs["mat"].Mul(enc_sparse).Decrypt(), values_m @ values1)
    plain_sparse = F.GetPlainVector(values1, EVectorFormat.sparse, scale)
    assert np.array_equal(objs["mat"].Mul(plain_sparse).Decrypt(), values_m @ values1)


def test_add_subtract_multiply(F, objs):
    e1, e2, p2 = objs["enc1"], objs["enc2"], objs["plain2"]
    assert np.array_equal(e1.Add(e2).Decrypt(), values1 + values2)
    assert np.array_equal(e1.Add(p2).Decrypt(), values1 + values2)
    assert np.array_equal(e1.Subtract(e2).Decrypt(), values1 - values2)
    assert np.array_equal(e1.Subtract(p2).Decrypt(), values1 - values2)
    assert np.array_equal(e1.PointwiseMultiply(e2).Decrypt(), values1 * values2)
    assert np.array_equal(e1.PointwiseMultiply(p2).Decrypt(), values1 * values2)


def test_dot_product_and_sum(F, objs):
    e1, e2, p2 = objs["enc1"], objs["enc2"], objs["plain2"]
    assert e1.DotProduct(e2).Decrypt()[0] == float(values1 @ values2)
    assert e1.DotProduct(p2).Decrypt()[0] == float(values1 @ values2)
    assert e1.SumAllSlots().Decrypt()[0] == values1.sum()
    # README.md:61-73 BasicExample: (1,2,3).(1,2,3) = 14, sum = 6, elementwise (1,2,3)*(-1,5,-4)
    from cryptonets_b200.interfaces import EVectorFormat
    a = F.GetEncryptedVector(np.array([1.0, 2, 3]), EVectorFormat.dense, 1)
    b = F.GetEncryptedVector(np.array([-1.0, 5, -4]), EVectorFormat.dense, 1)
    assert a.DotProduct(a).Decrypt()[0] == 14
    assert a.SumAllSlots().Decrypt()[0] == 6
    assert list(a.PointwiseMultiply(b).Decrypt()) == [-1, 10, -12]


def test_meta(F, objs):
    e1 = objs["enc1"]
    assert e1.IsEncrypted and not objs["plain2"].IsEncrypted
    assert e1.Scale == scale
    c = F.CopyVector(e1)
    c.RegisterScale(20)
    assert np.array_equal(c.Decrypt(), values1 * scale / 20)


@pytest.mark.parametrize("count", [4096 // 8, 10, 4096 // 8 - 5])
def test_duplicate(F, objs, count):
    dup = objs["enc1"].Duplicate(count)
    assert dup.Dim == count * 8
    d = dup.Decrypt()
    exp = np.zeros(8)
    exp[:6] = values1
    assert np.array_equal(d, np.tile(exp, count))


def test_packed_dot_products(F, objs):
    from cryptonets_b200.interfaces import EVectorFormat
    res = objs["enc1"].DotProduct(objs["enc2"], length=4).Decrypt()
    assert res[3] == float(values1[:4] @ values2[:4])
    rng = np.random.default_rng(5)
    data = np.rint(rng.normal(0, 1, 4096) * 10)
    enc = F.GetEncryptedVector(data, EVectorFormat.dense, 1)
    res = enc.DotProduct(enc, length=1024).Decrypt()
    for i in range(4):
        assert res[1024 * i + 1023] == float(data[i * 1024:(i + 1) * 1024] @ data[i * 1024:(i + 1) * 1024])


def test_interleave(F):
    from cryptonets_b200.interfaces import EMatrixFormat
    mat = np.array([[1, 0, 0, 2, 0, 0], [3, 0, 0, 4, 0, 0]], dtype=np.float64).T
    m = F.GetEncryptedMatrix(mat, EMatrixFormat.ColumnMajor, 10)
    assert list(m.Interleave(1).Decrypt()) == [1, 3, 0, 2, 4, 0]
    mat = np.array([[0, 0, 1, 0, 0, 2], [0, 0, 3, 0, 0, 4], [0, 0, 5, 0, 0, 6]], dtype=np.float64).T
    m = F.GetEncryptedMatrix(mat, EMatrixFormat.ColumnMajor, 10)
    assert list(m.Interleave(-1).Decrypt()) == [5, 3, 1, 6, 4, 2]


def test_permute(F):
    from cryptonets_b200.interfaces import EVectorFormat
    v = F.GetEncryptedVector(np.arange(1, 11, dtype=np.float64), EVectorFormat.dense, 1)
    s1, s2 = np.zeros(10), np.zeros(10)
    s1[[1, 4]] = 1
    s2[[3, 6]] = 1
    sel1, sel2 = F.GetPlainVector(s1, EVectorFormat.dense, 1), F.GetPlainVector(s2, EVectorFormat.dense, 1)
    w = v.Permute([sel1, sel2], [1, 2], 5)
    assert list(w.Decrypt()) == [2, 4, 0, 5, 7]


def test_big_stack(F):
    from cryptonets_b200.interfaces import EMatrixFormat, EVectorFormat
    n = 1050
    v = [F.GetEncryptedVector(np.arange(i * n, (i + 1) * n, dtype=np.float64), EVectorFormat.dense, 1) for i in range(4)]
    m = F.GetMatrix(v, EMatrixFormat.ColumnMajor)
    vec = m.ConvertToColumnVector()
    assert np.array_equal(vec.Decrypt(), np.arange(4 * n, dtype=np.float64))


def test_generate_value_from_string(F):
    primes = [40961, 65537, 114689, 147457, 188417]
    expected = [21399, 63588, 101610, 90324, 148561]
    v = F.GetValueFromString(",".join(str(x) for x in expected))
    assert [v % p for p in primes] == expected
    assert F.GetStringFromValue(v) == ",".join(str(x) for x in expected)


def test_rotate_matches_raw_semantics(F):
    from cryptonets_b200.interfaces import EVectorFormat
    from cryptonets_b200.raw import RawFactory
    vals = np.arange(1, 21, dtype=np.float64)
    enc = F.GetEncryptedVector(vals, EVectorFormat.dense, 1)
    raw = RawFactory(4096 // 2).GetEncryptedVector(vals, EVectorFormat.dense, 1)  # one batching row
    for amount in (1, 3, -2):
        got = enc.Rotate(amount).Decrypt()
        want = raw.Rotate(amount).Decrypt()
        assert np.array_equal(got, want), amount


def test_errors_mirror_reference(F, objs):
    from cryptonets_b200 import CnheError
    from cryptonets_b200.interfaces import EVectorFormat
    other = F.GetEncryptedVector(values1, EVectorFormat.dense, 7)
    with pytest.raises(CnheError, match="Scales do not match"):
        objs["enc1"].Add(other)
    short = F.GetEncryptedVector(values1[:3], EVectorFormat.dense, scale)
    with pytest.raises(CnheError, match="Dimensions do not match"):
        objs["enc1"].Add(short)
    with pytest.raises(CnheError, match="multiplying two plaintexts"):
        objs["plain2"].PointwiseMultiply(objs["plain2"])


@pytest.mark.parametrize("force_dense", [False, True])
def test_rowmajor_matrix_vector_batched_equals_per_row(F, force_dense):
    """LLDenseLayer's product (EncryptedSealBfvMatrix.cs:79-120): the batched device routine must give the very ciphertexts of the
    reference's per-row DotProduct loop, and the plain result."""
    from cryptonets_b200.interfaces import EMatrixFormat, EVectorFormat
    rng = np.random.default_rng(8)
    W = rng.integers(-9, 10, (7, 40)).astype(np.float64)
    x = rng.integers(-20, 21, 40).astype(np.float64)
    M = F.GetPlainMatrix(W, EMatrixFormat.RowMajor, 4)
    v = F.GetEncryptedVector(x, EVectorFormat.dense, 2)
    M.Batched = True
    a = M.Mul(v, None, force_dense)
    M.Batched = False
    b = M.Mul(v, None, force_dense)
    assert a.Dim == b.Dim == 7 and a.Scale == b.Scale == 8 and a.Format == b.Format
    got = a.Decrypt()
    assert np.array_equal(got[:7], W @ x)
    for ch in range(F.engine.P):
        for blk in range(a.vec.blocks):
            assert np.array_equal(a.vec.export_raw(ch, blk), b.vec.export_raw(ch, blk)), (ch, blk)


def test_pipelined_import_export_and_batched_dispose(F):
    """The serving-loop entry points: cnhe_vecs_import_raw on the upload stream (several imports in flight, slots rotating),
    cnhe_vecs_export_raw_async tickets waited out of order, cnhe_vecs_destroy.  Every batch must come back word for word, and the
    vectors imported from host words must decrypt to the values that were encrypted."""
    import torch
    eng = F.engine
    rng = np.random.default_rng(4)
    n = 6
    vals = rng.integers(-500, 500, (n, eng.N)).astype(np.float64)
    src = eng.encrypt_many(vals, 3.0)
    words = eng.export_raw_many(src)                                  # [P][n][1][ct_words], synchronous path
    host = torch.from_numpy(words.reshape(-1).astype(np.int64)).pin_memory()
    outs = [torch.zeros_like(host).pin_memory() for _ in range(4)]
    batches, tickets = [], []
    for i in range(4):                                                # 4 uploads queued back to back, none waited for
        vecs = eng.import_raw_many(host.data_ptr(), n, 1, eng.N, 3.0)
        batches.append(vecs)
        tickets.append(eng.export_raw_many_async(vecs, outs[i].data_ptr()))
    for i in (2, 0, 3, 1):
        eng.export_wait(tickets[i])
        assert torch.equal(outs[i], host), i
    from cryptonets_b200.he import B200BfvVector
    assert np.array_equal(B200BfvVector(F, batches[3][2]).Decrypt(), vals[2])
    for vecs in batches:
        eng.dispose_many(vecs)
        assert all(not v.h for v in vecs)
    eng.dispose_many(src)
    eng.dispose_many([])                                              # no-op
    again = eng.import_raw_many(host.data_ptr(), n, 1, eng.N, 3.0)    # slots are reusable after their release
    assert np.array_equal(eng.export_raw_many(again).reshape(-1), words.reshape(-1))
    eng.dispose_many(again)


def test_plain_columns_times_encrypted_scalars(F):
    """DenseMatrixBySparseVectorMultiply, third mode (AtomicSealBfvVector.cs:476-485): plain dense columns x an ENCRYPTED sparse vector --
    MultiplyPlain(sparse.enc[k], column k) per column, AddMany."""
    from cryptonets_b200.interfaces import EMatrixFormat, EVectorFormat
    m = np.array([[1, -2, 3], [4, 5, -6], [7, 8, 9], [-10, 11, 12]], dtype=np.float64)
    s = np.array([3, -4, 5], dtype=np.float64)
    pm = F.GetPlainMatrix(m, EMatrixFormat.ColumnMajor, 2)
    es = F.GetEncryptedVector(s, EVectorFormat.sparse, 3)
    out = pm.Mul(es)
    assert out.IsEncrypted and out.Scale == 6 and out.Dim == 4
    assert np.array_equal(np.asarray(out.Decrypt()), m @ s)
    # the same product with the roles swapped (encrypted columns x plain scalars) decrypts to the same values
    em = F.GetEncryptedMatrix(m, EMatrixFormat.ColumnMajor, 2)
    assert np.array_equal(np.asarray(em.Mul(F.GetPlainVector(s, EVectorFormat.sparse, 3)).Decrypt()), m @ s)


def test_permute_with_encrypted_selection_is_rejected_like_seal(F):
    """Permute's ct x ct branch (AtomicSealBfvVector.cs:1455-1458) multiplies WITHOUT relinearising and then rotates the size-3 product;
    SEAL 3.2's rotate_rows throws "encrypted size must be 2" on it, and so does the library."""
    from cryptonets_b200.interfaces import EVectorFormat
    v = F.GetEncryptedVector(np.arange(1, 11, dtype=np.float64), EVectorFormat.dense, 1)
    s1 = np.zeros(10)
    s1[[1, 4]] = 1
    enc_sel = F.GetEncryptedVector(s1, EVectorFormat.dense, 1)
    with pytest.raises(Exception, match="encrypted size must be 2"):
        v.Permute([enc_sel], [1], 5)


def test_concurrent_callers(F):
    """The reference calls the evaluator from up to ThreadCount threads at once (Utils.cs:68-86).  Four host threads hammer one context
    (serialised by its mutex) while a fifth drives a second context on the same GPU; every result must be exact."""
    import threading
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.interfaces import EVectorFormat
    rng = np.random.default_rng(7)
    data = [rng.integers(-50, 50, 64).astype(np.float64) for _ in range(4)]
    errors = []

    def worker(i, factory):
        try:
            a = data[i]
            for _ in range(6):
                e = factory.GetEncryptedVector(a, EVectorFormat.dense, 1)
                sq = e.PointwiseMultiply(e)
                tot = sq.Add(e).SumAllSlots()
                assert np.array_equal(np.asarray(sq.Decrypt()), a * a)
                assert tot.Decrypt()[0] == float((a * a + a).sum())
                for x in (e, sq, tot):
                    x.Dispose()
        except Exception as ex:  # pragma: no cover
            errors.append((i, repr(ex)))

    F2 = B200BfvFactory([40961, 65537], 4096, seed=3)
    try:
        threads = [threading.Thread(target=worker, args=(i, F)) for i in range(4)] + [threading.Thread(target=worker, args=(0, F2))]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    finally:
        F2.Dispose()
    assert not errors, errors


def test_big_integer_vectors_and_full_precision(F):
    """IFactory.GetEncryptedVector(IEnumerable<BigInteger>) / IVector.DecryptFullPrecision (IFactory.cs:43, EncryptedSealBfvVector.cs:188-199,
    343-348): values beyond 2^53 survive exactly (the product of the five default primes is ~2^81)."""
    from cryptonets_b200.interfaces import EVectorFormat
    big = [3 * 10 ** 20 + 7, -(2 ** 70) - 12345, 0, 999]
    e = F.GetEncryptedVector(big, EVectorFormat.dense)
    assert e.DecryptFullPrecision() == big
    p = F.GetPlainVector([5, -6, 7, 8], EVectorFormat.dense)
    prod = e.PointwiseMultiply(p)
    assert prod.DecryptFullPrecision() == [big[0] * 5, big[1] * -6, 0, 999 * 8]
    s = F.GetEncryptedVector([2 ** 60, -3], EVectorFormat.sparse)
    assert s.DecryptFullPrecision() == [2 ** 60, -3]
