"""Mul(DeferRelinearization=True) on the Raw backend and the deferred product's bindings: no GPU needed."""
import os
import re

import numpy as np
import pytest

from cryptonets_b200.interfaces import EMatrixFormat, EVectorFormat
from cryptonets_b200.raw import RawFactory

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_raw_mul_deferred_equals_mul():
    f = RawFactory(4096)
    rng = np.random.default_rng(1)
    m = rng.integers(-50, 50, (300, 17)).astype(np.float64)
    v = rng.integers(-50, 50, 17).astype(np.float64)
    M = f.GetEncryptedMatrix(m, EMatrixFormat.ColumnMajor, 2.0)
    V = f.GetEncryptedVector(v, EVectorFormat.sparse, 3.0)
    want, got = M.Mul(V), M.Mul(V, DeferRelinearization=True)
    assert np.array_equal(np.asarray(got.Decrypt()), np.asarray(want.Decrypt()))
    assert got.Scale == want.Scale == 6.0


def test_raw_mul_deferred_misuse_raises():
    f = RawFactory(4096)
    m = np.ones((8, 4))
    col = f.GetEncryptedMatrix(m, EMatrixFormat.ColumnMajor, 1.0)
    with pytest.raises(Exception, match="DeferRelinearization"):
        col.Mul(f.GetEncryptedVector(np.ones(4), EVectorFormat.dense, 1.0), DeferRelinearization=True)
    with pytest.raises(Exception, match="DeferRelinearization"):
        col.Mul(f.GetEncryptedVector(np.ones(4), EVectorFormat.sparse, 1.0), ForceDenseFormat=True, DeferRelinearization=True)
    with pytest.raises(Exception, match="DeferRelinearization"):
        f.GetEncryptedMatrix(m.T, EMatrixFormat.RowMajor, 1.0).Mul(f.GetEncryptedVector(np.ones(8), EVectorFormat.dense, 1.0),
                                                                   DeferRelinearization=True)


def test_entry_points_exported_declared_and_bound():
    from cryptonets_b200 import _lib
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "cnhe.h")).read()
    cs = open(os.path.join(ROOT, "integration", "B200Native.cs")).read()
    for name in ("cnhe_mat_mul_colmajor_sparse_deferred", "cnhe_context_product_sum_terms"):
        assert hasattr(L, name) and name in _lib.EXPORTS
        assert re.search(r"\bint %s\(" % name, header), name
        assert re.search(r"static extern int %s\(" % name, cs), name
    assert "public IVector MulDeferred(IVector v)" in cs


def test_csharp_bindings_check():
    import importlib.util
    spec = importlib.util.spec_from_file_location("check_csharp_bindings", os.path.join(ROOT, "tools", "check_csharp_bindings.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    errors, n = mod.check()
    assert not errors, errors
    assert n >= 113
