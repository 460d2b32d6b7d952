"""Enumerations of the reference plugin API (`HE Wrapper/IVector.cs:15-18`, `IMatrix.cs:14-17`)."""
import enum


class EVectorFormat(enum.IntEnum):
    dense = 0
    sparse = 1


class EMatrixFormat(enum.IntEnum):
    ColumnMajor = 0
    RowMajor = 1


def check_deferred_mul(m, v, force_dense, encrypted=True):
    """the cases Mul(DeferRelinearization=True) serves: a column-major matrix times a sparse vector, both encrypted (encrypted=False: a
    backend without ciphertexts checks the shapes only)"""
    if m.Format != EMatrixFormat.ColumnMajor or force_dense:
        raise Exception("DeferRelinearization applies to a column-major matrix times a sparse vector (without ForceDenseFormat)")
    if v.Format != EVectorFormat.sparse:
        raise Exception("DeferRelinearization expects a sparse vector")
    if encrypted and not (m.IsEncrypted and v.IsEncrypted):
        raise Exception("DeferRelinearization needs an encrypted matrix and an encrypted vector; Mul without it serves the other cases")
