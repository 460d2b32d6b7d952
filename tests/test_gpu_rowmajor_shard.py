"""cnhe_mat_mul_rowmajor_shard, the row-major product of a contiguous slice of the matrix rows (one rank's part of a dense layer split over
several GPUs): the slices' partial products must give the full product bit for bit, across the 1024-product waves of the full product and
with slice boundaries inside a wave; and its refusals."""
import numpy as np
import pytest

from cryptonets_b200._lib import CnheError

pytestmark = pytest.mark.gpu

ERR_INVALID = -1
T, N = 40961, 4096
ROWS = 1100                       # two waves of the full product: rows 0..1023 and 1024..1099
SLICES = [(0, 600), (600, 1050), (1050, 1100)]  # 600 and 1050 fall inside the full product's first and second wave


@pytest.fixture(scope="module")
def setup():
    from cryptonets_b200.engine import Engine
    eng = Engine([T], N, 10, 20, -1)
    eng.keygen(77)
    rng = np.random.default_rng(5)
    W = rng.integers(-1, 2, (ROWS, N)).astype(np.float64)
    x = rng.integers(-1, 2, N).astype(np.float64)
    rows = [eng.plain(r) for r in W]
    v = eng.encrypt(x)
    yield eng, W, x, rows, v
    eng.close()


def test_dense_slices_add_up_to_the_full_product(setup):
    """ForceDenseFormat: each slice's masks sit at its global columns, so the engine.add sum of the slices' outputs (modular addition is
    exact: the order does not matter) equals cnhe_mat_mul_rowmajor word for word."""
    eng, W, x, rows, v = setup
    full = eng.mat_mul_rowmajor(rows, v, force_dense=True)
    parts = [eng.mat_mul_rowmajor_shard(rows[a:b], v, True, a, ROWS) for a, b in SLICES]
    assert all(p.dim == ROWS and p.blocks == 1 for p in parts)
    acc = eng.add(parts[0], parts[1])
    total = eng.add(acc, parts[2])
    assert np.array_equal(eng.export_raw_many([total]), eng.export_raw_many([full]))
    assert np.array_equal(eng.decrypt(full), W @ x)
    eng.dispose_many(parts + [acc, total, full])


def test_sparse_slices_are_the_full_products_blocks(setup):
    """Sparse output: the slices' blocks laid end to end are the full product's blocks."""
    eng, W, x, rows, v = setup
    full = eng.mat_mul_rowmajor(rows, v, force_dense=False)
    parts = [eng.mat_mul_rowmajor_shard(rows[a:b], v, False, a, ROWS) for a, b in SLICES]
    assert [p.dim for p in parts] == [b - a for a, b in SLICES]
    got = np.concatenate([eng.export_raw_many([p]) for p in parts], axis=2)
    assert np.array_equal(got, eng.export_raw_many([full]))
    assert np.array_equal(eng.decrypt(full), W @ x)
    eng.dispose_many(parts + [full])


def test_refusals_leave_the_context_usable(setup):
    """A slice outside the matrix, more rows than slots for the dense output, and encrypted rows are CNHE_ERR_INVALID; the context keeps
    working afterwards."""
    eng, W, x, rows, v = setup
    enc_rows = [eng.encrypt(W[0]), eng.encrypt(W[1])]
    bad = [
        lambda: eng.mat_mul_rowmajor_shard(rows[:10], v, True, -1, 20),
        lambda: eng.mat_mul_rowmajor_shard(rows[:10], v, True, 15, 20),
        lambda: eng.mat_mul_rowmajor_shard(rows[:10], v, False, 0, 5),
        lambda: eng.mat_mul_rowmajor_shard(rows[:10], v, True, 0, N + 1),
        lambda: eng.mat_mul_rowmajor_shard(enc_rows, v, True, 0, 2),
    ]
    for i, call in enumerate(bad):
        with pytest.raises(CnheError) as e:
            call()
        assert e.value.code == ERR_INVALID, i
        ok = eng.mat_mul_rowmajor_shard(rows[2:4], v, False, 2, ROWS)
        assert np.array_equal(eng.decrypt(ok), W[2:4] @ x), i
        ok.dispose()
    eng.dispose_many(enc_rows)
