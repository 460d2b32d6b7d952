"""B200 backend of the CryptoNets plugin API: IFactory / IVector / IMatrix / IComputationEnvironment.

Python mirror of the C# shim a maintainer would add next to `EncryptedSealBfvFactory` (INTEGRATION.md): same member names,
argument meaning and exception behaviour as `HE Wrapper/IFactory.cs:20-130`, `IVector.cs:20-136`, `IMatrix.cs:18-122`, with
every method a call into libcnhe.so.  Vectors hold device handles instead of SEAL `Ciphertext[]`.
Errors surface as Python exceptions carrying the reference's message (the reference throws System.Exception)."""
import numpy as np

from .engine import ALL_SLOTS, Engine, Vec, _cuda_tensor
from .interfaces import EMatrixFormat, EVectorFormat, check_deferred_mul


class B200BfvEnvironment:
    """IComputationEnvironment (`HE Wrapper/IComputationEnvironment.cs:12-24`).  All environments of a factory share the
    context's CUDA stream; the object exists so that reference call sites keep their shape."""

    def __init__(self, factory):
        self.ParentFactory = factory

    Primes = property(lambda s: list(s.ParentFactory.engine.primes))


class B200BfvVector:
    """IVector over a device-resident cnhe_vec (== EncryptedSealBfvVector, `EncryptedSealBfvVector.cs:150-573`)."""

    def __init__(self, factory, vec):
        self.factory = factory
        self.vec = vec
        self.IsSigned = True

    eng = property(lambda s: s.factory.engine)
    Dim = property(lambda s: s.vec.dim)
    Scale = property(lambda s: s.vec.scale)
    Format = property(lambda s: EVectorFormat(s.vec.format))
    IsEncrypted = property(lambda s: s.vec.is_encrypted)
    BlockSize = property(lambda s: s.eng.N)
    Data = property(lambda s: s.vec)

    def _wrap(self, vec):
        return B200BfvVector(self.factory, vec)

    def Dispose(self):
        if self.vec is not None:
            self.vec.dispose()
            self.vec = None

    def Write(self, writer):
        """IVector.Write(StreamWriter) (`EncryptedSealBfvVector.cs:428-437`)."""
        writer.write(self.eng.write_vector(self.vec))

    def RegisterScale(self, scale):
        self.vec.register_scale(scale)

    def RegisterDim(self, dim):
        self.vec.register_dim(dim)

    def Decrypt(self, env=None, device=False):
        """The values as numpy, or with device=True (or a torch device) as a CUDA tensor (Engine.decrypt_many)."""
        if device is not False:
            return self.eng.decrypt_many([self.vec], device=device)[0]
        return self.eng.decrypt(self.vec)

    def DecryptFullPrecision(self, env=None):
        """IVector.DecryptFullPrecision (`EncryptedSealBfvVector.cs:343-348,397-411`): exact integers (Python ints stand in for BigInteger),
        the CRT join of the per-modulus residues, centred when the vector is signed; NOT divided by Scale (the reference does not)."""
        f, res = self.factory, self.eng.decrypt_residues(self.vec)
        out = []
        for j in range(res.shape[1]):
            x = sum(int(c) * int(res[i, j]) for i, c in enumerate(f.preComputedCoefficients)) % f.bigFactor
            if self.IsSigned and x * 2 > f.bigFactor:
                x -= f.bigFactor
            out.append(x)
        return out

    def Add(self, v, env=None):
        return self._wrap(self.eng.add(self.vec, v.vec))

    def Subtract(self, v, env=None):
        return self._wrap(self.eng.sub(self.vec, v.vec))

    def PointwiseMultiply(self, v, env=None):
        return self._wrap(self.eng.pointwise_multiply(self.vec, v.vec))

    def DotProduct(self, v, env=None, length=None, ForceOutputInColumn=None):
        fc = -1 if ForceOutputInColumn is None else ForceOutputInColumn
        return self._wrap(self.eng.dot_product(self.vec, v.vec, ALL_SLOTS if length is None else length, fc))

    def SumAllSlots(self, env=None, length=None, ForceOutputInColumn=None):
        fc = -1 if ForceOutputInColumn is None else ForceOutputInColumn
        return self._wrap(self.eng.sum_all_slots(self.vec, ALL_SLOTS if length is None else length, fc))

    def Duplicate(self, count, env=None):
        return self._wrap(self.eng.duplicate(self.vec, count))

    def Rotate(self, amount, env=None):
        return self._wrap(self.eng.rotate(self.vec, amount))

    def Permute(self, selections, shifts, outputDim, env=None):
        sel = [None if s is None else s.vec for s in selections]
        return self._wrap(self.eng.permute(self.vec, sel, shifts, outputDim))



def _poly_layer(engine, vecs, a, b, c):
    """PolyActivation's call: the quadratic (a, b, c) through cnhe_layer_poly2, or a = 4 or 5 coefficient vectors, highest degree first,
    through cnhe_layer_poly"""
    v = lambda x: None if x is None else x.vec
    if isinstance(a, (list, tuple)):
        if b is not None or c is not None:
            raise Exception("a list of coefficients takes no b or c")
        return engine.layer_poly(vecs, [v(x) for x in reversed(a)])
    return engine.layer_poly2(vecs, a.vec, v(b), v(c))

class B200BfvMatrix:
    """IMatrix as an array of vectors (`HE Wrapper/EncryptedSealBfvMatrix.cs:14-231`)."""

    def __init__(self, factory, vectors, fmt=EMatrixFormat.ColumnMajor, CopyVectors=True):
        if vectors and any(v.Dim != vectors[0].Dim for v in vectors):
            raise Exception("all columns of a matrix should have the same size")
        self.factory = factory
        self.vectors = [factory.CopyVector(v) for v in vectors] if CopyVectors else list(vectors)
        self.Format = fmt
        self.DataDisposedExternaly = False
        self.Batched = True  # False replays the reference's per-row call sequence

    eng = property(lambda s: s.factory.engine)
    RowCount = property(lambda s: len(s.vectors) if s.Format == EMatrixFormat.RowMajor else s.vectors[0].Dim)
    ColumnCount = property(lambda s: len(s.vectors) if s.Format == EMatrixFormat.ColumnMajor else s.vectors[0].Dim)
    Scale = property(lambda s: s.vectors[0].Scale)
    BlockSize = property(lambda s: s.eng.N)
    IsEncrypted = property(lambda s: all(v.IsEncrypted for v in s.vectors))
    Data = property(lambda s: s.vectors)

    def Write(self, writer):
        """IMatrix.Write(StreamWriter) (`EncryptedSealBfvMatrix.cs:199-208`)."""
        nl = "\r\n"
        writer.write("<Start LargeEncryptedMatrix>" + nl + EMatrixFormat(self.Format).name + nl + str(len(self.vectors)) + nl)
        for v in self.vectors:
            v.Write(writer)
        writer.write("<End LargeEncryptedMatrix>" + nl)

    def Dispose(self):
        if self.vectors is not None and not self.DataDisposedExternaly:
            vs = [v for v in self.vectors if v is not None and v.vec is not None]
            if vs:
                self.eng.dispose_many([v.vec for v in vs])
            for v in vs:
                v.vec = None
        self.vectors = None

    def RegisterScale(self, scale):
        for v in self.vectors:
            v.RegisterScale(scale)

    def Decrypt(self, env=None, device=False):
        """The values as numpy, or with device=True (or a torch device) as a CUDA tensor in the same orientation (Engine.decrypt_many)."""
        rows = self.eng.decrypt_many([v.vec for v in self.vectors], device=device)
        return rows if self.Format == EMatrixFormat.RowMajor else rows.T

    def MulRows(self, v, ForceDenseFormat, first_row, total_rows):
        """Row-major product for a slice of the rows held by this matrix (global rows first_row..): the per-rank piece of a row-sharded
        dense layer (cnhe_mat_mul_rowmajor_shard; cryptonets_b200/parallel.py combines the pieces)."""
        if self.Format != EMatrixFormat.RowMajor:
            raise Exception("MulRows expects a RowMajor matrix")
        return B200BfvVector(self.factory, self.eng.mat_mul_rowmajor_shard([r.vec for r in self.vectors], v.vec, ForceDenseFormat, first_row, total_rows))

    def Mul(self, v, env=None, ForceDenseFormat=False, DeferRelinearization=False):
        """DeferRelinearization (B200-specific, column-major encrypted matrix times an encrypted sparse vector only): sum the products
        before relinearising, one relinearisation per output block (Engine.mat_mul_colmajor_sparse_deferred); same decrypted values"""
        f = self.factory
        if DeferRelinearization:
            check_deferred_mul(self, v, ForceDenseFormat)
            return B200BfvVector(f, self.eng.mat_mul_colmajor_sparse_deferred([c.vec for c in self.vectors], v.vec))
        if self.Format == EMatrixFormat.ColumnMajor:
            if ForceDenseFormat:
                raise Exception("Forcing dense format is available only in RowMajor mode")
            return B200BfvVector(f, self.eng.mat_mul_colmajor_sparse([c.vec for c in self.vectors], v.vec))
        if self.Batched and v.IsEncrypted and not self.IsEncrypted and v.vec.blocks == 1:
            # all rows through each stage together (same ciphertexts as the per-row loop below)
            return B200BfvVector(f, self.eng.mat_mul_rowmajor([r.vec for r in self.vectors], v.vec, ForceDenseFormat))
        if not ForceDenseFormat:  # EncryptedSealBfvMatrix.cs:79-89
            tmp = [row.DotProduct(v, env) for row in self.vectors]
            res = B200BfvVector(f, self.eng.generate_sparse_of_array([t.vec for t in tmp]))
            for t in tmp:
                t.Dispose()
            return res
        total = None  # EncryptedSealBfvMatrix.cs:90-120
        for i, row in enumerate(self.vectors):
            t = row.DotProduct(v, env, ForceOutputInColumn=i)
            if total is None:
                total = t
            else:
                s = total.Add(t, env)
                total.Dispose()
                t.Dispose()
                total = s
        total.RegisterDim(len(self.vectors))
        if total.Format != EVectorFormat.dense:
            raise Exception("Internal probloem: expecting the output to be dense")
        return total

    def PrepareDiagonal(self, baby_steps=0, ntt_bytes=0, fold_width=None):
        """This plain row-major matrix prepared for the diagonal (baby-step / giant-step) product, B200BfvFactory.MulDiagonalBatch; the
        rows stay owned by this matrix.  baby_steps = 0 picks the number of baby steps with the fewest key switches.  ntt_bytes: device
        memory to spend on holding diagonals in NTT form (Engine.diag_prepare; 0 none, None all), same products, faster.  fold_width: None
        for the generalised diagonals, else the folded product for few rows (0 lets the library choose the width)."""
        if self.Format != EMatrixFormat.RowMajor:
            raise Exception("the diagonal product expects a RowMajor matrix")
        return B200BfvDiagonalMatrix(self.factory, self.eng.diag_prepare([r.vec for r in self.vectors], baby_steps, ntt_bytes, fold_width))

    def _check(self, m):
        if m.Format != self.Format:
            raise Exception("Format mismatch")
        if m.RowCount != self.RowCount:
            raise Exception("Row count mismatch")
        if m.ColumnCount != self.ColumnCount:
            raise Exception("Column count mismatch")

    def Add(self, m, env=None):
        self._check(m)
        out = [a.Add(b, env) for a, b in zip(self.vectors, m.vectors)]
        return B200BfvMatrix(self.factory, out, self.Format, CopyVectors=False)

    def ElementWiseMultiply(self, m, env=None):
        self._check(m)
        if m is self:  # SquareActivation: one batched wave over every column
            out = self.eng.layer_square([v.vec for v in self.vectors])
            return B200BfvMatrix(self.factory, [B200BfvVector(self.factory, o) for o in out], self.Format, CopyVectors=False)
        out = [a.PointwiseMultiply(b, env) for a, b in zip(self.vectors, m.vectors)]
        return B200BfvMatrix(self.factory, out, self.Format, CopyVectors=False)

    def PolyActivation(self, a, b=None, c=None, env=None):
        """a x^2 + b x + c of every column in one wave (cnhe_layer_poly2): a, b, c plain sparse vectors of dimension 1 at scales W, W s and
        W s^2 (b, c may be None); the result has scale W s^2.  a may instead be a sequence of 4 or 5 such vectors, highest degree first
        (None for 0, the first required), for the cubic or quartic of cnhe_layer_poly (b and c then None): coefficient j at scale
        W s^(d - j), the result at scale W s^d."""
        out = _poly_layer(self.eng, [v.vec for v in self.vectors], a, b, c)
        return B200BfvMatrix(self.factory, [B200BfvVector(self.factory, o) for o in out], self.Format, CopyVectors=False)

    def GetColumn(self, i):
        if i >= len(self.vectors):
            raise Exception("Column does not exist")
        if self.Format != EMatrixFormat.ColumnMajor:
            raise Exception("Columns can be extracted only from a column major matrix")
        return self.vectors[i]

    def GetRow(self, i):
        if i >= len(self.vectors):
            raise Exception("Row does not exist")
        if self.Format != EMatrixFormat.RowMajor:
            raise Exception("Rows can be extracted only from a row major matrix")
        return self.vectors[i]

    def SetColumn(self, i, vector):
        if i >= len(self.vectors):
            raise Exception("Column does not exist")
        if self.Format != EMatrixFormat.ColumnMajor:
            raise Exception("Columns can be set only from a column major matrix")
        if vector.Dim != self.vectors[i].Dim:
            raise Exception("dimension of vector does not match the dimension of the vector it is replacing")
        if vector.Scale != self.vectors[i].Scale:
            raise Exception("Scale of vector does not match the scale of the vector it is replacing")
        if vector.IsEncrypted != self.vectors[i].IsEncrypted:
            raise Exception("can't exchange encrypted and not encrypted vectors")
        self.vectors[i] = vector

    def ConvertToColumnVector(self, env=None):
        return B200BfvVector(self.factory, self.eng.stack([v.vec for v in self.vectors]))

    def Interleave(self, shift, env=None):
        if self.Format != EMatrixFormat.ColumnMajor:
            raise Exception("Expecting ColumnMajor matrix")
        return B200BfvVector(self.factory, self.eng.interleave([v.vec for v in self.vectors], shift))


class B200BfvDiagonalMatrix:
    """A plain matrix held as its pre-rotated generalised diagonals on the device (include/cnhe.h, cnhe_diag_prepare)."""

    def __init__(self, factory, diag):
        self.factory = factory
        self.diag = diag

    def Info(self):
        return self.diag.info()

    def NttInfo(self):
        return self.diag.ntt_info()

    def FoldWidth(self):
        return self.diag.fold_width()

    def ExportNtt(self, channel, index):
        return self.diag.export_ntt(channel, index)

    RowCount = property(lambda s: s.diag.info()["n_rows"])
    ColumnCount = property(lambda s: s.diag.info()["dim"])

    def Dispose(self):
        if self.diag is not None:
            self.diag.dispose()
            self.diag = None


def _read_block(reader, end_marker):
    """lines of a text stream up to and including the line `end_marker`"""
    out = []
    while True:
        line = reader.readline()
        if not line:
            raise Exception("Bad stream format.")
        out.append(line)
        if line.rstrip("\r\n") == end_marker:
            return "".join(out)


class B200BfvFactory:
    """IFactory (`HE Wrapper/IFactory.cs:20-130`); constructor arguments of EncryptedSealBfvFactory (`:247-260`)."""

    DefaultDecompositionBitCount = 10
    DefaultGaloisDecompositionBitCount = 20

    def __init__(self, primes=None, n=4096, DecompositionBitCount=10, GaloisDecompositionBitCount=20, SmallModulusCount=-1, seed=None,
                 device=0, generate_keys=True):
        """seed=None (default): keys and encryption randomness from the OS CSPRNG, as SEAL's KeyGenerator/Encryptor give the reference.
        An integer seed selects the deterministic sampler shared with the CPU oracle: parity tests only."""
        if isinstance(primes, (str, bytes, bytearray)):  # EncryptedSealBfvFactory(fileName) (IFactory.cs:262-265): parameters and keys from a key archive
            data = open(primes, "rb").read() if isinstance(primes, str) else bytes(primes)
            if data[:4] == b"CNHK":  # a compact key blob (SaveCompactKeys): keys expanded on the GPU, no secret key
                self.engine = Engine(None, compact_keys=data, device=device)
            else:
                self.engine = Engine(None, archive=data, device=device)
            primes = self.engine.primes
        else:
            if primes is None:
                primes, n = [40961, 65537, 114689, 147457, 188417], 4096  # IFactory.cs:247-253
            self.engine = Engine(primes, n, DecompositionBitCount, GaloisDecompositionBitCount, SmallModulusCount, device)
            if generate_keys:
                self.engine.keygen(seed)
        self._env = B200BfvEnvironment(self)
        big = 1
        for p in primes:
            big *= int(p)
        self.bigFactor = big
        self.preComputedCoefficients = [(big // int(p)) * pow((big // int(p)) % int(p), -1, int(p)) for p in primes]

    Primes = property(lambda s: list(s.engine.primes))

    def AllocateComputationEnv(self):
        return self._env

    def FreeComputationEnv(self, env):
        pass

    def _big(self, v, fmt, encrypt):  # the IEnumerable<BigInteger> overloads (IFactory.cs:29,43): SplitBigNumbers on exact integers
        vals = [int(x) % self.bigFactor for x in v]
        res = np.array([[x % int(p) for x in vals] for p in self.engine.primes], dtype=np.uint64)
        return B200BfvVector(self, self.engine.from_residues(res, 1.0, int(fmt), encrypt))

    def GetPlainVector(self, v, fmt, scale=None):
        if scale is None:
            return self._big(v, fmt, False)
        return B200BfvVector(self, self.engine.plain(np.asarray(v, dtype=np.float64), scale, int(fmt)))

    def GetEncryptedVector(self, v, fmt, scale=None):
        if scale is None:
            return self._big(v, fmt, True)
        return B200BfvVector(self, self.engine.encrypt(np.asarray(v, dtype=np.float64), scale, int(fmt)))

    def CopyVector(self, v):
        return B200BfvVector(self, self.engine.copy(v.vec))

    def _rows(self, m, fmt):
        """The vectors of matrix m as rows [n][dim]: a CUDA torch tensor stays on its device (transposed and made contiguous there)."""
        if _cuda_tensor(m):
            return m.T.contiguous() if fmt == EMatrixFormat.ColumnMajor else m
        m = np.asarray(m, dtype=np.float64)
        return m.T if fmt == EMatrixFormat.ColumnMajor else m

    def GetPlainMatrix(self, m, fmt, scale):
        vecs = [self.GetPlainVector(r, EVectorFormat.dense, scale) for r in self._rows(m, fmt)]
        return B200BfvMatrix(self, vecs, fmt, CopyVectors=False)

    def GetEncryptedMatrix(self, m, fmt, scale):
        """m: a numpy-compatible matrix or a CUDA torch tensor (encrypted from device memory)."""
        rows = self._rows(m, fmt)
        rows = rows if _cuda_tensor(rows) else np.ascontiguousarray(rows)
        vecs = [B200BfvVector(self, v) for v in self.engine.encrypt_many(rows, scale)]
        return B200BfvMatrix(self, vecs, fmt, CopyVectors=False)

    def GetEncryptedMatrixCompact(self, m, fmt, scale):
        """The same encryption as GetEncryptedMatrix as one compact blob (bytes) for a server: bit-packed c0 and per-channel ChaCha20 keys
        for c1 (include/cnhe.h, cnhe_vecs_encrypt_compact).  Needs the secret key; the matrix format travels out of band."""
        rows = self._rows(m, fmt)
        return self.engine.encrypt_compact(rows if _cuda_tensor(rows) else np.ascontiguousarray(rows), scale)

    def LoadCompactMatrix(self, data, fmt, slot=0):
        """The matrix of a compact blob (GetEncryptedMatrixCompact), expanded on the GPU; `fmt` is the format it was made with.  slot: the
        key slot (AddClientKeys) of the client that encrypted it."""
        vs = self.engine.import_compact(data)
        if slot:
            for v in vs:
                v.set_key_slot(slot)
        return B200BfvMatrix(self, [B200BfvVector(self, v) for v in vs], fmt, CopyVectors=False)

    # ---- several clients in one context (include/cnhe.h, key slots)
    def AddClientKeys(self, blob):
        """Another client's compact evaluation keys (its SaveCompactKeys; same parameters) in a new key slot; returns the slot."""
        return self.engine.add_client_compact(blob)

    def RemoveClient(self, slot):
        self.engine.remove_client(slot)

    def SquareBatch(self, matrices):
        """SquareActivation of several matrices (possibly of different clients) in one relinearisation wave."""
        vecs = [v.vec for m in matrices for v in m.vectors]
        out, i, res = self.engine.layer_square(vecs), 0, []
        for m in matrices:
            n = len(m.vectors)
            res.append(B200BfvMatrix(self, [B200BfvVector(self, o) for o in out[i:i + n]], m.Format, CopyVectors=False))
            i += n
        return res

    def PolyActivationBatch(self, matrices, a, b=None, c=None):
        """m.PolyActivation(a, b, c) of several matrices (possibly of different clients) in one relinearisation wave."""
        vecs = [v.vec for m in matrices for v in m.vectors]
        out = _poly_layer(self.engine, vecs, a, b, c)
        i, res = 0, []
        for m in matrices:
            n = len(m.vectors)
            res.append(B200BfvMatrix(self, [B200BfvVector(self, o) for o in out[i:i + n]], m.Format, CopyVectors=False))
            i += n
        return res

    def StackBatch(self, matrices):
        """ConvertToColumnVector of several column-major matrices (one per client) in one pass."""
        return [B200BfvVector(self, o) for o in self.engine.stack_many([[v.vec for v in m.vectors] for m in matrices])]

    def ConvBatch(self, matrices, weights):
        """[m.Mul(w) for w in weights] for every column-major matrix m (one per client, same shape) in one scalar-MAC call: the
        clients' columns side by side, output (b, k) gathering client b's columns with weights[k]."""
        B, K = len(matrices), len(matrices[0].vectors)
        if any(len(m.vectors) != K for m in matrices) or any(w.Dim != K for w in weights):
            raise Exception("dimensions do not match")
        M = B * len(weights)
        gather = [b * K + kk for b in range(B) for _ in weights for kk in range(K)]
        out = self.engine.layer_conv_dense([v.vec for m in matrices for v in m.vectors], gather, [w.vec for _ in range(B) for w in weights], None, M, K)
        n = len(weights)
        return [[B200BfvVector(self, o) for o in out[b * n:(b + 1) * n]] for b in range(B)]

    def MulRowMajorBatch(self, weights, vectors, ForceDenseFormat=False):
        """weights.Mul(v, ForceDenseFormat=...) of a plain row-major matrix for every v (one per client) in one pass."""
        out = self.engine.mat_mul_rowmajor_batch([r.vec for r in weights.vectors], [v.vec for v in vectors], ForceDenseFormat)
        return [B200BfvVector(self, o) for o in out]

    def DuplicateBatch(self, vectors, count):
        """v.Duplicate(count) for every encrypted vector (one per client; key slots may differ) in one pass."""
        return [B200BfvVector(self, o) for o in self.engine.duplicate_many([v.vec for v in vectors], count)]

    def PermuteBatch(self, vector_list, selections, shifts, outputDim):
        """[v.Permute(selections[j], shifts[j], outputDim) for j] for every encrypted vector (one per client) in one pass; one list of
        permuted vectors per client."""
        perms = [([None if s is None else s.vec for s in sel], sh) for sel, sh in zip(selections, shifts)]
        out, P = self.engine.permute_many([v.vec for v in vector_list], perms, outputDim), len(perms)
        return [[B200BfvVector(self, o) for o in out[b * P:(b + 1) * P]] for b in range(len(vector_list))]

    def DotRowsBatch(self, weights, vectors, length=None):
        """[weights.GetRow(r).DotProduct(v, length=length) for r] of a plain row-major matrix for every v (one per client) in one pass; one
        list of products per client."""
        R = len(weights.vectors)
        out = self.engine.dot_rows_batch([r.vec for r in weights.vectors], [v.vec for v in vectors], ALL_SLOTS if length is None else length)
        return [[B200BfvVector(self, o) for o in out[b * R:(b + 1) * R]] for b in range(len(vectors))]

    def InterleaveBatch(self, matrices, shift):
        """m.Interleave(shift) of several column-major matrices (one per client, same column count) in one pass."""
        return [B200BfvVector(self, o) for o in self.engine.interleave_many([[v.vec for v in m.vectors] for m in matrices], shift)]

    def MultiplyPlainBatch(self, vectors, plain):
        """v.PointwiseMultiply(plain) for every encrypted vector and one plain dense vector in one pass."""
        return [B200BfvVector(self, o) for o in self.engine.multiply_plain_many([v.vec for v in vectors], plain.vec)]

    def MulDiagonalBatch(self, diag, vectors):
        """diag (B200BfvMatrix.PrepareDiagonal) times every encrypted vector (one per client; key slots may differ) in one pass; each result
        decrypts to the matrix's Mul(v, ForceDenseFormat=True)."""
        return [B200BfvVector(self, o) for o in self.engine.mat_mul_diagonal(diag.diag, [v.vec for v in vectors])]

    def GetMatrix(self, vectors, fmt, CopyVectors=True):
        return B200BfvMatrix(self, vectors, fmt, CopyVectors=CopyVectors)

    # ---- levels (include/cnhe.h, cnhe_context_derive_level; DESIGN 4.17)
    CoeffModulusCount = property(lambda s: s.engine.k)

    def AtLevel(self, k):
        """The factory of this one's level on its first k coefficient primes (the restriction of its keys and key slots), made once and
        cached; k equal to this factory's count is the factory itself."""
        if k == self.engine.k:
            return self
        levels = self.__dict__.setdefault("_levels", {})
        if k not in levels:
            f = B200BfvFactory.__new__(B200BfvFactory)
            f.engine = self.engine.derive_level(k)
            f._env = B200BfvEnvironment(f)
            f.bigFactor, f.preComputedCoefficients = self.bigFactor, self.preComputedCoefficients
            levels[k] = f
        return levels[k]

    def ModSwitch(self, m, level_factory):
        """An encrypted matrix or vector of this factory switched to level_factory (AtLevel), every ciphertext on fewer primes."""
        return self.ModSwitchBatch([m], level_factory)[0]

    def ModSwitchBatch(self, items, level_factory):
        """ModSwitch of several matrices or vectors (possibly of different clients) in one pass."""
        vecs = [v.vec for it in items for v in (it.vectors if isinstance(it, B200BfvMatrix) else [it])]
        out, i, res = self.engine.mod_switch(vecs, level_factory.engine), 0, []
        for it in items:
            if isinstance(it, B200BfvMatrix):
                n = len(it.vectors)
                res.append(B200BfvMatrix(level_factory, [B200BfvVector(level_factory, o) for o in out[i:i + n]], it.Format, CopyVectors=False))
            else:
                n = 1
                res.append(B200BfvVector(level_factory, out[i]))
            i += n
        return res

    # ---- sanitisation (include/cnhe.h, cnhe_vecs_sanitize; DESIGN 4.18)
    def SanitizeMaxBits(self):
        """The widest flood width Sanitize accepts, floor(log2(q/t)) - 2."""
        return self.engine.sanitize_max_bits()

    def Sanitize(self, m, flood_bits):
        """An encrypted matrix or vector re-randomised under its key slot's public key with a flood of flood_bits bits in its noise: what
        a result should be before it goes back to its client."""
        return self.SanitizeBatch([m], flood_bits)[0]

    def SanitizeBatch(self, items, flood_bits):
        """Sanitize of several matrices or vectors (possibly of different clients) in one pass."""
        vecs = [v.vec for it in items for v in (it.vectors if isinstance(it, B200BfvMatrix) else [it])]
        out, i, res = self.engine.sanitize(vecs, flood_bits), 0, []
        for it in items:
            if isinstance(it, B200BfvMatrix):
                n = len(it.vectors)
                res.append(B200BfvMatrix(self, [B200BfvVector(self, o) for o in out[i:i + n]], it.Format, CopyVectors=False))
            else:
                n = 1
                res.append(B200BfvVector(self, out[i]))
            i += n
        return res

    # ---- wire formats (IFactory.cs:474-495; SEAL streams unpinned, see csrc/wire.cu)
    def Save(self, target, withPrivateKeys=False):
        """IFactory.Save(stream | fileName, withPrivateKeys): the ZIP key archive."""
        data = self.engine.save_keys(withPrivateKeys)
        if isinstance(target, str):
            with open(target, "wb") as f:
                f.write(data)
        else:
            target.write(data)
        return target

    def SaveCompactKeys(self, target=None, public=True, relin=True, galois=None):
        """The evaluation keys a server needs as one compact blob (include/cnhe.h, cnhe_keys_save_compact): a freshly generated key set under
        this factory's secret key, `a` of every key regenerated on the server's GPU from a per-channel ChaCha20 key, `b` bit-packed.
        galois: None = every standard element, [] = none (CryptoNets never rotates), else the elements the network rotates by.  Returns the
        bytes, or writes them to `target` (file name or binary stream); B200BfvFactory(blob or file name) is the server side."""
        data = self.engine.save_compact_keys(public, relin, galois)
        if target is None:
            return data
        if isinstance(target, str):
            with open(target, "wb") as f:
                f.write(data)
        else:
            target.write(data)
        return target

    def LoadVector(self, reader):
        """IFactory.LoadVector(StreamReader): `reader` is a text stream positioned at "<Start LargeEncryptedVector>"."""
        text = _read_block(reader, "<End LargeEncryptedVector>")
        vec, _ = self.engine.read_vector(text)
        return B200BfvVector(self, vec)

    def LoadMatrix(self, reader):  # EncryptedSealBfvMatrix.Read (EncryptedSealBfvMatrix.cs:182-197)
        if reader.readline().rstrip("\r\n") != "<Start LargeEncryptedMatrix>":
            raise Exception("Bad stream format.")
        fmt = EMatrixFormat[reader.readline().strip()]
        n = int(reader.readline())
        vecs = [self.LoadVector(reader) for _ in range(n)]
        if reader.readline().rstrip("\r\n") != "<End LargeEncryptedMatrix>":
            raise Exception("Bad stream format.")
        return B200BfvMatrix(self, vecs, fmt, CopyVectors=False)

    def GetValueFromString(self, s):  # IFactory.cs:395-403
        f = [int(x) for x in s.split(",")]
        return sum(c * x for c, x in zip(self.preComputedCoefficients, f)) % self.bigFactor

    def GetStringFromValue(self, value):
        return ",".join(str(int(value) % int(p)) for p in self.engine.primes)

    # fused layer entry point used by PoolLayer.Apply (NeuralNetworks/PoolLayer.cs:149-229)
    def ConvDenseLayer(self, inputs, gather, weights, bias, M, K):
        out = self.engine.layer_conv_dense([v.vec for v in inputs], gather, [w.vec for w in weights],
                                           None if bias is None else [b.vec for b in bias], M, K)
        return [B200BfvVector(self, o) for o in out]

    def ActivationConvDenseLayer(self, inputs, a, b, c, gather, weights, bias, M, K):
        """PoolLayer(DeferRelinearization=True) over its activation's input: the activation (a, b, c None: the square; else PolyActivation's
        quadratic) and ConvDenseLayer in one call, relinearising the M outputs instead of every squared input."""
        v = lambda x: None if x is None else x.vec
        out = self.engine.layer_activation_conv_dense([x.vec for x in inputs], v(a), v(b), v(c), gather, [w.vec for w in weights],
                                                      None if bias is None else [x.vec for x in bias], M, K)
        return [B200BfvVector(self, o) for o in out]

    def CaptureInference(self, net, example_inputs, SpanLevels=False):
        """Records the layers of `net` after its EncryptLayer once, on example_inputs, as one CUDA graph (include/cnhe.h,
        cnhe_capture_begin): a CapturedInference whose Run(inputs) replays the whole chain with one launch.  example_inputs is one encrypted
        input matrix (the network's GetNext path, Apply per layer) or a list of them, one per client, each bound to its client's key slot
        (the serve_batch path, ApplyBatch per layer).  The chain runs once eagerly on the examples first, so that the layers build their
        long-lived state outside the graph.  Runs must use the same shapes, scales and key slots; the network's prepared weights
        and the factory's keys are read in place and must outlive the capture.  The example matrices become the graph's inputs: every Run
        writes its inputs' words into them, so they belong to the capture until it is disposed.  Run serves any client of the factory: it
        binds the graph's key switches to the key slots its inputs carry (include/cnhe.h, cnhe_graph_bind).
        SpanLevels: a network built with levels= records across the level factories its ModSwitchLayers run on (level_factories,
        include/cnhe.h cnhe_capture_begin_levels); the outputs are then matrices of the lowest level.  Without it, a chain that switches
        levels is refused (CNHE_ERR_STATE)."""
        return CapturedInference(self, net, example_inputs, SpanLevels)

    def Dispose(self):
        for f in self.__dict__.get("_levels", {}).values():
            f.Dispose()
        self.engine.close()


def level_factories(chain):
    """The level factories the ModSwitchLayers of `chain` (a network's layers after its EncryptLayer) run on, in chain order, each once:
    the contexts a recording of the chain enlists (CaptureInference(SpanLevels=True)).  A switch on a factory without levels (RawFactory)
    passes its matrix through and names none."""
    from .layers import BaseLayer, ModSwitchLayer
    out = []
    for layer in chain:
        if isinstance(layer, ModSwitchLayer):
            f = layer.Factory
            if f is not BaseLayer.Factory.fget(layer) and not any(f is g for g in out):
                out.append(f)
    return out


def graph_binding(positions, recorded, current):
    """The slots to bind a recorded graph's key positions to (include/cnhe.h, cnhe_graph_bind): input vector j was recorded in key slot
    recorded[j] and its replacement belongs to slot current[j], so position recorded[j] is bound to current[j].  A position no input was
    recorded in keeps its own slot.  Raises when one recorded slot would be bound to two slots."""
    to = {}
    for r, c in zip(recorded, current):
        if to.setdefault(r, c) != c:
            raise Exception("the inputs bind recorded key slot %d to two key slots (%d and %d)" % (r, to[r], c))
    return [to.get(p, p) for p in positions]


class CapturedInference:
    """One inference of a network recorded as a CUDA graph (B200BfvFactory.CaptureInference).  The example input matrices are the graph's
    inputs (Run overwrites them with its inputs' words, one device copy per matrix and plaintext prime when each matrix's vectors lie in
    one slab, as encrypted and imported matrices do); the output matrices the recording made are graph-owned: their words are those of
    the latest Run and valid until the next one.  TimingLayers are left out: they time and synchronise the host, which a replay does
    not do."""

    def __init__(self, factory, net, example_inputs, SpanLevels=False):
        from .layers import EncryptLayer, TimingLayer
        self.factory, self.graph, self.outputs = factory, None, None
        self.batch = isinstance(example_inputs, (list, tuple))
        examples = list(example_inputs) if self.batch else [example_inputs]
        chain, layer = [], net
        while not isinstance(layer, EncryptLayer):
            if not isinstance(layer, TimingLayer):
                chain.append(layer)
            layer = layer.Source
        chain.reverse()
        for layer in chain:
            if not layer.layerPrepared:
                layer.Prepare()
                layer.layerPrepared = True
        self.inputs = examples
        # the key slot of every example vector as recorded: Run binds each to the slot of the input vector that takes its place
        self.recorded_slots = [v.vec.key_slot for m in examples for v in m.vectors]
        eng = factory.engine
        # One eager pass first: layers build long-lived state (bias vectors, scalar-MAC plans) on their first Apply.  Built while recording,
        # it would sit in graph memory that holds no words until a launch -- and never, if the recording is refused -- and later eager
        # inferences of the network would read it.
        for m in self._apply(chain, examples):
            m.Dispose()
        # the level factories exist after the eager pass, and hold the restriction of every key slot the examples carry
        eng.capture_begin(levels=[f.engine for f in level_factories(chain)] if SpanLevels else None)
        try:
            ms = self._apply(chain, examples)
            self.graph = eng.capture_end()
        except BaseException:
            eng.capture_abort()
            raise
        self.outputs = ms
        self.positions = self.graph.slots()  # the graph's key positions, and the slots they are bound to
        self.bound = list(self.positions)

    def _apply(self, chain, inputs):
        """the layers on the input matrices, each intermediate disposed once read (as serve_batch and GetNext do: while recording, later
        recorded allocations reuse its memory); the inputs are kept"""
        ms = list(inputs)
        try:
            for layer in chain:
                out = layer.ApplyBatch(ms) if self.batch else [layer.Apply(ms[0])]
                for m, o in zip(ms, out):
                    if o is not m and not any(m is i for i in inputs):
                        m.Dispose()
                ms = out
        except BaseException:
            for m in ms:
                if not any(m is i for i in inputs):
                    m.Dispose()
            raise
        return ms

    def Info(self):
        """dict(kernel_nodes, device_bytes) of the recorded graph."""
        return self.graph.info()

    def Run(self, inputs):
        """Assigns `inputs` (shaped as the example inputs: one matrix, or a list of one per client) to the recorded inputs, launches the
        graph and returns the output matrix (or list of them).  Asynchronous like any other call; reading the outputs orders after it.
        The inputs may belong to other clients than the examples did: the graph is bound to their key slots (graph_binding) and the outputs
        report them.  Inputs that would bind one recorded key slot to two clients, or that a bind or the assignment refuses, leave the
        graph's binding and the recorded inputs' key slots as they were."""
        ms = list(inputs) if self.batch else [inputs]
        if len(ms) != len(self.inputs) or any(len(m.vectors) != len(i.vectors) for m, i in zip(ms, self.inputs)):
            raise Exception("the inputs are not shaped as the recorded ones")
        eng = self.factory.engine
        src = [v.vec for m in ms for v in m.vectors]
        dst = [v.vec for m in self.inputs for v in m.vectors]
        slots = [v.key_slot for v in src]
        binding = graph_binding(self.positions, self.recorded_slots, slots)
        tags = [d.key_slot for d in dst]
        self.graph.bind(binding)
        try:
            for d, s in zip(dst, slots):
                if d.key_slot != s:
                    d.set_key_slot(s)
            eng.vecs_assign(dst, src)
        except BaseException:
            # a refused assignment leaves the graph's binding and the recorded inputs' key slots as they were (as far as the slots they
            # were bound to still exist)
            try:
                self.graph.bind(self.bound)
                for d, t in zip(dst, tags):
                    if d.key_slot != t:
                        d.set_key_slot(t)
            except Exception:  # noqa: BLE001 -- the assignment's error is the one to report
                pass
            raise
        self.bound = binding
        self.graph.launch()
        return list(self.outputs) if self.batch else self.outputs[0]

    def Dispose(self):
        """Releases the outputs and the graph; the example input matrices stay the caller's."""
        for m in self.outputs or []:
            m.Dispose()
        self.outputs = None
        if self.graph is not None:
            self.graph.dispose()
            self.graph = None
