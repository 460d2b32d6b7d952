"""Raw (plaintext) backend: the reference's own fake backend over doubles, restated with numpy.

Mirrors `HE Wrapper/RawVector.cs:14-268`, `RawMatrix.cs:12-174` and `RawFactory` (`IFactory.cs:138-238`).  The reference uses
it as the source of EncryptLayer's input matrices, as the mock for layer tests, and as the semantic model every decrypted
result is compared with; it plays the same three roles here.  It is not a fallback of the encrypted path."""
import numpy as np

from .interfaces import EMatrixFormat, EVectorFormat, check_deferred_mul
from .engine import _cuda_tensor


def _round(a):
    return np.rint(np.asarray(a, dtype=np.float64))  # Math.Round: ties to even


class RawEnvironment:
    def __init__(self, factory):
        self.ParentFactory = factory
        self.Primes = getattr(factory, "Primes", None)


class RawVector:
    Max = 0.0

    def __init__(self, v, scale, block_size, fmt=EVectorFormat.dense):
        v = np.atleast_1d(np.asarray(v, dtype=np.float64))
        if np.isinf(v).any():
            raise Exception("infinity")
        self.Scale = scale
        self.v = _round(v * scale)
        self.BlockSize = block_size
        self.Format = fmt
        self.IsSigned = True

    @classmethod
    def _of(cls, values, scale, block_size, fmt=EVectorFormat.dense):
        o = cls(values, 1, block_size, fmt)
        o.Scale = scale
        return o

    Dim = property(lambda s: 0 if s.v is None else len(s.v))
    Data = property(lambda s: s.v.copy())
    IsEncrypted = property(lambda s: False)

    def Dispose(self):
        self.v = None

    def RegisterScale(self, scale):
        self.Scale = scale

    def Decrypt(self, env=None):
        RawVector.Max = max(RawVector.Max, float(np.abs(self.v).max()))
        return self.v / self.Scale

    def Add(self, v, env=None):
        if self.Scale == 0:
            return v
        if v.Scale == 0:
            return self
        if self.Scale != v.Scale:
            raise Exception("Scales do not match.")
        return RawVector._of(self.v + v.v, self.Scale, self.BlockSize)

    def Subtract(self, v, env=None):
        if v.Scale == 0:
            return self
        if self.Scale != 0 and self.Scale != v.Scale:
            raise Exception("Scales do not match.")
        return RawVector._of(self.v - v.v, self.Scale, self.BlockSize)

    def PointwiseMultiply(self, v, env=None):
        if len(self.v) == len(v.v):
            mul = self.v * v.v
        elif len(self.v) == 1 and self.Format == EVectorFormat.sparse:
            mul = v.v * self.v[0]
        elif len(v.v) == 1 and v.Format == EVectorFormat.sparse:
            mul = self.v * v.v[0]
        else:
            raise Exception("Vectors dimensions do not match")
        return RawVector._of(mul, self.Scale * v.Scale, self.BlockSize)

    @staticmethod
    def _rot(w, length, n):
        res = np.zeros(n)
        if len(w) > n - length:
            res[length:] = w[: n - length]
            res[: len(w) - (n - length)] = w[n - length:]
        else:
            res[length: length + len(w)] = w
        return res

    def DotProduct(self, w, env=None, length=None):
        if length is None:
            return RawVector._of([float(np.dot(self.v, w.v))], self.Scale * w.Scale, self.BlockSize)
        res = self.v * w.v
        skip = 1
        while skip < length:  # RawVector.cs:166-182
            res = res + RawVector._rot(res, skip, self.Dim)
            skip *= 2
        return RawVector._of(res, self.Scale * w.Scale, self.BlockSize)

    def SumAllSlots(self, env=None):
        return RawVector._of([float(self.v.sum())], self.Scale, self.BlockSize)

    def Duplicate(self, count, env=None):
        shift = 1
        while shift < self.Dim:
            shift *= 2
        w = np.zeros(shift * count)
        for i in range(count):
            w[i * shift: i * shift + self.Dim] = self.v
        return RawVector(w / self.Scale, self.Scale, self.BlockSize)

    def _rotate_values(self, vec, amount):
        n = len(self.v)
        w = np.zeros(n)
        for i in range(len(vec)):
            k = (i + amount) % self.BlockSize
            if k < n:
                w[i] = vec[k]
        return w

    def Rotate(self, amount, env=None):
        return RawVector._of(self._rotate_values(self.v, amount), self.Scale, self.BlockSize)

    def Permute(self, selections, shifts, outputDim, env=None):
        if len(selections) != len(shifts):
            raise Exception("number of selection vectors and number of shifts does not match")
        res = np.zeros(self.Dim)
        for s, sh in zip(selections, shifts):
            if s is None:
                continue
            if s.Dim != self.Dim:
                raise Exception("dimension of selection vector does not match dimension of data vector")
            res = res + self._rotate_values(self.v * s.v, sh)
        return RawVector._of(res[:outputDim], self.Scale * selections[0].Scale, self.BlockSize)



def poly_scale(W, s, e):
    """W s^e with the powers of s multiplied up one factor at a time, as cnhe_layer_poly forms the scales it checks"""
    r = W
    for _ in range(e):
        r *= s
    return r

class RawMatrix:
    Max = 0.0

    def __init__(self, m, scale, fmt, block_size):
        """m: a numpy-compatible matrix, or a CUDA torch tensor (an input matrix that stays on its device: its Data is a tensor, which an
        encrypting factory reads from device memory; the Raw backend's own operations take numpy matrices)"""
        self.Scale = scale
        self.Format = fmt
        if _cuda_tensor(m):
            import torch
            self.m = torch.round(m.to(torch.float64) * scale)  # ties to even, as np.rint
        else:
            self.m = _round(np.asarray(m, dtype=np.float64) * scale)
        self.BlockSize = block_size
        self.DataDisposedExternaly = False

    RowCount = property(lambda s: s.m.shape[0])
    ColumnCount = property(lambda s: s.m.shape[1])
    Data = property(lambda s: s.m.clone() if _cuda_tensor(s.m) else s.m.copy())
    IsEncrypted = property(lambda s: False)

    def Dispose(self):
        self.m = None

    def RegisterScale(self, scale):
        self.Scale = scale

    def Decrypt(self, env=None):
        return self.m / self.Scale

    def Mul(self, v, env=None, ForceDenseFormat=False, DeferRelinearization=False):
        """DeferRelinearization changes nothing in exact arithmetic; the shapes the encrypted backend refuses with it are refused here too"""
        if DeferRelinearization:
            check_deferred_mul(self, v, ForceDenseFormat, encrypted=False)
        return RawVector._of(self.m @ v.v, self.Scale * v.Scale, v.BlockSize)

    def _check(self, m):
        if m.Format != self.Format:
            raise Exception("Format mismatch")
        if m.RowCount != self.RowCount:
            raise Exception("Row count mismatch")
        if m.ColumnCount != self.ColumnCount:
            raise Exception("Column count mismatch")

    def ElementWiseMultiply(self, m, env=None):
        self._check(m)
        r = RawMatrix(self.m * m.m, 1, self.Format, m.BlockSize)
        r.Scale = self.Scale * m.Scale
        return r

    def PolyActivation(self, a, b=None, c=None, env=None):
        """A x^2 + B x + C on every scaled integer: a, b, c are sparse vectors of dimension 1 at scales W, W s, W s^2 (b, c may be None),
        checked exactly as cnhe_layer_poly2 checks them.  a may instead be a sequence of 4 or 5 coefficient vectors, highest degree first
        (None for 0, the first required), checked as cnhe_layer_poly checks them: the integer polynomial, evaluated exactly."""
        if isinstance(a, (list, tuple)):
            if b is not None or c is not None:
                raise Exception("a list of coefficients takes no b or c")
            return self._poly(a)
        out_scale = a.Scale * self.Scale * self.Scale
        if (b is not None and b.Scale * self.Scale != out_scale) or (c is not None and c.Scale != out_scale):
            raise Exception("Scales do not match.")
        r = RawMatrix(a.v[0] * self.m * self.m, 1, self.Format, self.BlockSize)
        if b is not None:
            r.m = r.m + b.v[0] * self.m
        if c is not None:
            r.m = r.m + c.v[0]
        r.Scale = out_scale
        return r

    def _poly(self, coeffs):
        d = len(coeffs) - 1
        if d not in (3, 4):
            raise Exception("the degree must be 3 or 4")
        if coeffs[0] is None:
            raise Exception("the leading coefficient is required")
        s, W = self.Scale, coeffs[0].Scale
        for i, v in enumerate(coeffs[1:], 1):  # coefficient of x^(d - i), at scale W s^i
            if v is not None and v.Scale != poly_scale(W, s, i):
                raise Exception("Scales do not match.")
        x = self.m.astype(np.int64).astype(object)  # exact integers: the polynomial's terms may pass 2^53
        acc = np.full(x.shape, int(coeffs[0].v[0]), dtype=object)
        for v in coeffs[1:]:
            acc = acc * x + (0 if v is None else int(v.v[0]))
        r = RawMatrix(np.zeros(self.m.shape), 1, self.Format, self.BlockSize)
        r.m = np.array(acc.tolist(), dtype=np.float64).reshape(self.m.shape)
        r.Scale = poly_scale(W, s, d)
        return r

    def Add(self, m, env=None):
        self._check(m)
        if m.Scale != self.Scale:
            raise Exception("Scale mismatch")
        r = RawMatrix(self.m + m.m, 1, self.Format, m.BlockSize)
        r.Scale = self.Scale
        return r

    def GetColumn(self, i):
        if i >= self.ColumnCount:
            raise Exception("Column does not exist")
        if self.Format != EMatrixFormat.ColumnMajor:
            raise Exception("Columns can be extracted only from a column major matrix")
        return RawVector._of(self.m[:, i], self.Scale, self.BlockSize)

    def GetRow(self, i):
        if i >= self.RowCount:
            raise Exception("Row does not exist")
        if self.Format != EMatrixFormat.RowMajor:
            raise Exception("Row can be extracted only from a row major matrix")
        return RawVector._of(self.m[i, :], self.Scale, self.BlockSize)

    def SetColumn(self, i, vector):
        self.m[:, i] = vector.v

    def ConvertToColumnVector(self, env=None):
        if self.ColumnCount * self.RowCount > self.BlockSize:
            raise Exception("block too long for interleaving")
        return RawVector._of(self.m.T.reshape(-1), self.Scale, self.BlockSize)  # MathNet Enumerate(): column major

    def Interleave(self, shift, env=None):
        if shift == 0:
            raise Exception("number of items cannot be zero")

        def sh(v, s):
            w = np.zeros(len(v))
            if s < 0:
                w[: len(v) + s] = v[-s:]
            else:
                w[s:] = v[: len(v) - s]
            return w

        w = self.m[:, 0].copy()
        for i in range(1, self.ColumnCount):
            w = w + sh(self.m[:, i], shift * i)
        return RawVector._of(w, self.Scale, self.BlockSize)


class RawFactory:
    def __init__(self, BlockSize=8192):
        self.BlockSize = BlockSize
        self.Primes = None
        self._env = None

    def GetPlainVector(self, v, fmt, scale):
        return RawVector(v, scale, self.BlockSize, fmt)

    GetEncryptedVector = GetPlainVector

    def CopyVector(self, v):
        return RawVector._of(v.v.copy(), v.Scale, v.BlockSize, v.Format)

    def GetPlainMatrix(self, m, fmt, scale):
        return RawMatrix(m, scale, fmt, self.BlockSize)

    GetEncryptedMatrix = GetPlainMatrix

    def GetMatrix(self, vectors, fmt, CopyVectors=True):
        scale = vectors[0].Scale
        cols = np.stack([v.v / scale for v in vectors], axis=1)
        return RawMatrix(cols, scale, fmt, self.BlockSize)

    def AllocateComputationEnv(self):
        if self._env is None:
            self._env = RawEnvironment(self)
        return self._env

    def FreeComputationEnv(self, env):
        pass

    def GetValueFromString(self, s):
        return int(s)

    def GetStringFromValue(self, value):
        return str(value)
