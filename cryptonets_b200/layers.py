"""Layer API of the reference (`NeuralNetworks/`), restated over the IFactory / IMatrix / IVector interfaces.

Same class and property names as the C# layer library so that the network definitions of `CryptoNets/CryptoNets.cs:20-75`
and `LowLatencyCryptoNets/LoLaCryptonets.cs:280-329` read the same.  Layers talk only to the plugin interfaces; with a
B200BfvFactory, PoolLayer.Apply issues one fused device call for the whole layer instead of the reference's per-output
fan-out (`PoolLayer.cs:196-227`), with identical outputs; pass Fused=False to replay the reference's call sequence."""
import time

import numpy as np

from .interfaces import EMatrixFormat, EVectorFormat
from .raw import RawFactory, RawMatrix, poly_scale


class ConvolutionEngine:
    """Index arithmetic of `NeuralNetworks/ConvolutionEngine.cs:10-145`."""

    def __init__(self):
        self.InputShape = None
        self._kernel = None
        self.Stride = None
        self.Padding = None
        self.Upperpadding = None
        self.Lowerpadding = None
        self.MapCount = None
        self.Offsets = None
        self.Corners = None
        self.prepared = False

    @property
    def KernelShape(self):
        return self._kernel

    @KernelShape.setter
    def KernelShape(self, value):
        self._kernel = list(value)
        offs, off = [], [0] * len(value)
        while True:  # first axis fastest (:39-54)
            offs.append(list(off))
            go = False
            for i in range(len(value)):
                off[i] += 1
                if off[i] < value[i]:
                    go = True
                    break
                off[i] = 0
            if not go:
                break
        self.Offsets = offs

    def Prepare(self):
        if self.prepared:
            return
        n = len(self.InputShape)
        self.Upperpadding = self.Upperpadding or [0] * n
        self.Lowerpadding = self.Lowerpadding or [0] * n
        self.Padding = self.Padding or [False] * n
        self.maps = int(np.prod(self.MapCount)) if self.MapCount is not None else 1
        ks = self._kernel
        lo = [-self.Lowerpadding[i] - (-(ks[i] // 2) if self.Padding[i] else 0) for i in range(n)]
        hi = [self.InputShape[i] + self.Upperpadding[i] - (((ks[i] + 1) // 2) if self.Padding[i] else ks[i]) for i in range(n)]
        corners, cur = [], list(lo)
        while True:  # last axis fastest (:61-79)
            corners.append(list(cur))
            go = False
            for i in range(n - 1, -1, -1):
                cur[i] += self.Stride[i]
                if cur[i] <= hi[i]:
                    go = True
                    break
                cur[i] = lo[i]
            if not go:
                break
        self.Corners = corners
        self.prepared = True

    def Location(self, corner, offset, shape, bias=0):
        if not self.prepared:
            self.Prepare()
        index = 0
        for i in range(len(offset)):
            cord = (corner[i] + offset[i]) if corner is not None else offset[i]
            if cord < 0 or cord >= shape[i]:
                return -1
            index = index * shape[i] + cord
        return index + bias

    def GetDenseWeights(self, weights):  # :121-144
        """The convolution as a dense [maps*corners x prod(InputShape)] row-major matrix (CIFAR: 5488 x 16268), vectorised."""
        self.Prepare()
        weights = np.asarray(weights, dtype=np.float64)
        shape = np.asarray(self.InputShape)
        nc, cols = len(self.Corners), int(np.prod(self.InputShape))
        ksize = int(np.prod(self._kernel))
        offs = np.asarray(self.Offsets)                                      # [O, n]
        coords = np.asarray(self.Corners)[:, None, :] + offs[None, :, :]      # [C, O, n]
        valid = np.all((coords >= 0) & (coords < shape), axis=2)
        loc = np.zeros(coords.shape[:2], dtype=np.int64)
        kidx = np.zeros(len(offs), dtype=np.int64)
        for i in range(len(shape)):                                          # same row-major index as Location()
            loc = loc * shape[i] + coords[:, :, i]
            kidx = kidx * self._kernel[i] + offs[:, i]
        ci, oi = np.nonzero(valid)
        mat = np.zeros((self.maps * nc, cols))
        for m in range(self.maps):
            mat[m * nc + ci, loc[ci, oi]] = weights[kidx[oi] + m * ksize]
        return mat.reshape(-1)

    def GetDenseBias(self, bias):
        return np.repeat(np.asarray(bias, dtype=np.float64)[: self.maps], len(self.Corners))


class BaseLayer:
    """`NeuralNetworks/BaseLayer.cs:9-105` (pull model: GetNext() asks the Source, then applies this layer)."""

    def __init__(self, **kw):
        self.Source = None
        self._factory = None
        self.Verbose = False
        self.layerPrepared = False
        self.LastSeconds = None
        for k, v in kw.items():
            setattr(self, k, v)

    @property
    def Factory(self):
        return self._factory if self._factory is not None else self.Source.Factory

    @Factory.setter
    def Factory(self, f):
        self._factory = f

    def Apply(self, m):
        raise NotImplementedError

    def ApplyBatch(self, ms):
        """Apply to one matrix per client (one inference each; on a multi-client factory their key slots may differ).  Layers without a
        batched form apply one matrix at a time; the outputs are the same either way."""
        return [self.Apply(m) for m in ms]

    def GetNext(self):
        if not self.layerPrepared:
            self.Prepare()
            self.layerPrepared = True
        m = self.Source.GetNext()
        start = time.time()
        res = self.Apply(m)
        self.LastSeconds = time.time() - start
        if self.Verbose:
            print("Layer %s computed in %.4f seconds layer width (%d,%d)" % (type(self).__name__, self.LastSeconds, m.RowCount, m.ColumnCount))
        if res is not m:
            m.Dispose()
        return res

    def GetOutputScale(self):
        return self.Source.GetOutputScale()

    def OutputDimension(self):
        return self.Source.OutputDimension()

    def Prepare(self):
        pass

    def PrepareNetwork(self):
        if self.Source is not None:
            self.Source.PrepareNetwork()
        self.Prepare()
        self.layerPrepared = True

    def DisposeNetwork(self):
        if self.Source is not None:
            self.Source.DisposeNetwork()
        self.Dispose()

    def Dispose(self):
        pass


class MatrixSource(BaseLayer):
    """Input layer over an in-memory feature matrix: the role of `BatchReader` (`BatchReader.cs:59-109`) with the TSV parsing
    replaced by a synthetic / caller-supplied array (no dataset ships with the reference).  rows = images."""

    def __init__(self, features, Scale=1.0, NormalizationFactor=1.0, MaxSlots=None, labels=None):
        super().__init__()
        self.features = np.asarray(features, dtype=np.float64)
        self.Scale = Scale
        self.NormalizationFactor = NormalizationFactor
        self.MaxSlots = MaxSlots or len(self.features)
        self.Labels = labels
        self._factory = RawFactory(8192)
        self.pos = 0

    def PrepareNetwork(self):
        pass

    def DisposeNetwork(self):
        pass

    def GetNext(self):
        if self.pos >= len(self.features):
            self.pos = 0
        chunk = self.features[self.pos: self.pos + self.MaxSlots]
        self.pos += self.MaxSlots
        return RawMatrix(chunk * self.NormalizationFactor, self.Scale, EMatrixFormat.ColumnMajor, 0)

    def GetOutputScale(self):
        return self.Scale

    def OutputDimension(self):
        return self.features.shape[1]


class LLConvReader(MatrixSource):
    """One image -> im2col matrix [corners x offsets] (`LLConvReader.cs:96-158`)."""

    def __init__(self, features, Scale, NormalizationFactor, InputShape, KernelShape, Stride, Upperpadding=None, Lowerpadding=None, Padding=None):
        super().__init__(features, Scale, NormalizationFactor, MaxSlots=1)
        self.ce = ConvolutionEngine()
        self.ce.InputShape, self.ce.KernelShape, self.ce.Stride = InputShape, KernelShape, Stride
        self.ce.Upperpadding, self.ce.Lowerpadding, self.ce.Padding = Upperpadding, Lowerpadding, Padding
        self.ce.Prepare()

    def GetNext(self):
        if self.pos >= len(self.features):
            self.pos = 0
        f = self.features[self.pos] * self.NormalizationFactor
        self.pos += 1
        ce = self.ce
        mat = np.zeros((len(ce.Corners), len(ce.Offsets)))
        for c, corner in enumerate(ce.Corners):
            for o, off in enumerate(ce.Offsets):
                l = ce.Location(corner, off, ce.InputShape)
                mat[c, o] = f[l] if l >= 0 else 0
        return RawMatrix(mat, self.Scale, EMatrixFormat.ColumnMajor, 0)

    def OutputDimension(self):
        return len(self.ce.Corners)


class EncryptLayer(BaseLayer):
    """`NeuralNetworks/EncryptLayer.cs:10-20`"""

    def Apply(self, m):
        res = self.Factory.GetEncryptedMatrix(m.Data, EMatrixFormat.ColumnMajor, 1)
        res.RegisterScale(m.Scale)
        return res


class TimingLayer(BaseLayer):
    """`NeuralNetworks/TimingLayer.cs:15-66`; device work is asynchronous, so a counter boundary synchronises the factory first."""

    TotalTimeMS, N, StartTime = {}, {}, {}

    def __init__(self, StartCounters=(), StopCounters=(), **kw):
        super().__init__(**kw)
        self.StartCounters, self.StopCounters = list(StartCounters), list(StopCounters)

    @classmethod
    def Reset(cls):
        cls.TotalTimeMS.clear(); cls.N.clear(); cls.StartTime.clear()

    @classmethod
    def GetStats(cls):
        return "\t".join("%s %.2f" % (k, v / cls.N[k]) for k, v in cls.TotalTimeMS.items())

    def Apply(self, m):
        eng = getattr(self.Factory, "engine", None)
        if eng is not None:
            eng.sync()
        now = time.time()
        for c in self.StartCounters:
            TimingLayer.StartTime[c] = now
        for c in self.StopCounters:
            if c in TimingLayer.StartTime:
                TimingLayer.TotalTimeMS[c] = TimingLayer.TotalTimeMS.get(c, 0.0) + (now - TimingLayer.StartTime[c]) * 1000.0
                TimingLayer.N[c] = TimingLayer.N.get(c, 0) + 1
        return m


class SquareActivation(BaseLayer):
    """`NeuralNetworks/SquareActivation.cs:8-20`"""

    def Apply(self, m):
        return m.ElementWiseMultiply(m, self.Factory.AllocateComputationEnv())

    def ApplyBatch(self, ms):
        batch = getattr(self.Factory, "SquareBatch", None)
        if batch is None or len(ms) < 2:
            return super().ApplyBatch(ms)
        return batch(ms)

    def GetOutputScale(self):
        s = self.Source.GetOutputScale()
        return s * s


class PolyActivation(BaseLayer):
    """Quadratic activation a x^2 + b x + c (a learned polynomial such as a fitted ReLU or Swish) on every element.  Coefficients = (a, b,
    c), CoefficientScale = W: the integer coefficients are A = round(a W), B = round(b W s), C = round(c W s^2) for the input scale s,
    and the output scale is W s^2.  On a B200BfvFactory the whole layer is one call (cnhe_layer_poly2) with the square's passes; a
    coefficient that rounds to 0 is left out.  Slots: a dense vector's padding slots (beyond its dimension) stay zero, as they do for
    SquareActivation, so that rotating layers such as LLDuplicateLayer see only the data; each ciphertext of a sparse vector gets C in all
    of its slots (there the slots are separate images, which no layer mixes).

    Coefficients of length 4 or 5, (c_d, ..., c_0) highest degree first, give the cubic or quartic of cnhe_layer_poly (two levels of
    squares): coefficient j is round(c_j W s^(d - j)) and the output scale is W s^d.  c_d must not round to 0 mod any plaintext prime; the
    output scale grows as s^d, so the plaintext primes must hold the largest |value| below half their product."""

    def __init__(self, **kw):
        self.Coefficients = (1.0, 0.0, 0.0)
        self.CoefficientScale = 1.0
        self.coefficientVectors = None
        super().__init__(**kw)

    def Prepare(self):
        cs = [float(x) for x in self.Coefficients]
        if len(cs) not in (3, 4, 5):
            raise Exception("PolyActivation takes 3, 4 or 5 coefficients")
        W, s = self.CoefficientScale, self.Source.GetOutputScale()
        f = self.Factory

        def vec(v, scale):
            return None if np.rint(v * scale) == 0 else f.GetPlainVector([v], EVectorFormat.sparse, scale)

        if len(cs) == 3:
            a, b, c = cs
            self.coefficientVectors = (f.GetPlainVector([a], EVectorFormat.sparse, W), vec(b, W * s), vec(c, W * s * s))
        else:
            self.coefficientVectors = tuple([f.GetPlainVector([cs[0]], EVectorFormat.sparse, W)] +
                                            [vec(v, poly_scale(W, s, i)) for i, v in enumerate(cs[1:], 1)])

    def _args(self):
        # the quadratic's (a, b, c), or the cubic's / quartic's coefficient list
        return self.coefficientVectors if len(self.coefficientVectors) == 3 else (list(self.coefficientVectors),)

    def Apply(self, m):
        return m.PolyActivation(*self._args(), env=self.Factory.AllocateComputationEnv())

    def ApplyBatch(self, ms):
        batch = getattr(self.Factory, "PolyActivationBatch", None)
        if batch is None or len(ms) < 2:
            return super().ApplyBatch(ms)
        return batch(ms, *self._args())

    def GetOutputScale(self):
        s = self.Source.GetOutputScale()
        if len(self.Coefficients) == 3:
            return self.CoefficientScale * s * s
        return poly_scale(self.CoefficientScale, s, len(self.Coefficients) - 1)

    def Dispose(self):
        for v in self.coefficientVectors or ():
            if v is not None and hasattr(v, "Dispose"):
                v.Dispose()
        self.coefficientVectors = None


class _ConvLayerBase(BaseLayer):
    def __init__(self, **kw):
        self.ce = ConvolutionEngine()
        self.Weights = None
        self.Bias = None
        self.WeightsScale = 1.0
        self.weightWindows = None
        self.biasVectors = None
        self.kernelSize = -1
        super().__init__(**kw)

    InputShape = property(lambda s: s.ce.InputShape, lambda s, v: setattr(s.ce, "InputShape", list(v)))
    KernelShape = property(lambda s: s.ce.KernelShape, lambda s, v: setattr(s.ce, "KernelShape", list(v)))
    Stride = property(lambda s: s.ce.Stride, lambda s, v: setattr(s.ce, "Stride", list(v)))
    Padding = property(lambda s: s.ce.Padding, lambda s, v: setattr(s.ce, "Padding", list(v)))
    Upperpadding = property(lambda s: s.ce.Upperpadding, lambda s, v: setattr(s.ce, "Upperpadding", list(v)))
    Lowerpadding = property(lambda s: s.ce.Lowerpadding, lambda s, v: setattr(s.ce, "Lowerpadding", list(v)))
    MapCount = property(lambda s: s.ce.MapCount, lambda s, v: setattr(s.ce, "MapCount", list(v)))
    Offsets = property(lambda s: s.ce.Offsets)
    Corners = property(lambda s: s.ce.Corners)

    def maps(self):
        return int(np.prod(self.MapCount)) if self.MapCount is not None else 1

    def GetOutputScale(self):
        return (len(self.Offsets) if self.Weights is None else self.WeightsScale) * self.Source.GetOutputScale()

    def _weight(self, offset, bias):
        l = self.ce.Location(None, offset, self.KernelShape, bias)
        return 0.0 if l < 0 else self.Weights[l]

    def PrepareWeightsWindows(self):  # PoolLayer.cs:101-111
        self.weightWindows = []
        for m in range(self.maps()):
            w = [self._weight(off, m * self.kernelSize) for off in self.Offsets]
            self.weightWindows.append(self.Factory.GetPlainVector(np.array(w), EVectorFormat.sparse, self.WeightsScale))

    def _bias_value(self, mapIndex):
        return self.Bias[mapIndex] if self.Bias is not None else self.Weights[(mapIndex + 1) * self.kernelSize - 1]

    def Dispose(self):
        for lst in (self.weightWindows, self.biasVectors):
            if lst:
                for v in lst:
                    if v is not None:
                        v.Dispose()
        self.weightWindows = self.biasVectors = None

    def OutputDimension(self):
        if not self.layerPrepared:
            self.Prepare()
        return len(self.Corners) * (1 if self.Weights is None else self.maps())


class PoolLayer(_ConvLayerBase):
    """Convolution / dense / mean-pool over per-pixel ciphertexts (`NeuralNetworks/PoolLayer.cs:13-245`).

    DeferRelinearization=True (with Fused, weights, and a SquareActivation or 3-coefficient PolyActivation as Source): GetNext takes the
    activation's input and makes one factory call (ActivationConvDenseLayer) that squares, sums the unrelinearised products and
    relinearises only this layer's outputs -- the same decryption with one key switch per output instead of one per input.  Apply and
    ApplyBatch are unchanged, and a factory without that call (the Raw backend) applies the activation, then this layer."""

    def __init__(self, Fused=True, DeferRelinearization=False, **kw):
        self.Fused = Fused
        self.DeferRelinearization = DeferRelinearization
        super().__init__(**kw)

    def Prepare(self):
        if self.DeferRelinearization:
            src = self.Source
            if not self.Fused:
                raise Exception("DeferRelinearization needs the fused layer (Fused=True)")
            if self.Weights is None:
                raise Exception("DeferRelinearization needs a layer with weights")
            if not isinstance(src, (SquareActivation, PolyActivation)):
                raise Exception("DeferRelinearization needs a SquareActivation or PolyActivation as Source")
            if isinstance(src, PolyActivation) and len(src.Coefficients) != 3:
                raise Exception("DeferRelinearization takes a quadratic PolyActivation (3 coefficients)")
        if self.layerPrepared:
            return
        self.ce.Prepare()
        self.kernelSize = int(np.prod(self.KernelShape)) + (1 if self.Bias is None else 0)
        if self.Weights is None:
            return
        self.PrepareWeightsWindows()
        self.biasVectors = None
        self.layerPrepared = True

    def _gather_row(self, corner):
        return [self.ce.Location(corner, off, self.InputShape) for off in self.Offsets]

    def GetNext(self):
        f = self.Factory
        if not (self.DeferRelinearization and hasattr(f, "ActivationConvDenseLayer")):
            return super().GetNext()
        act = self.Source
        for layer in (self, act):
            if not layer.layerPrepared:
                layer.Prepare()
                layer.layerPrepared = True
        m = act.Source.GetNext()
        start = time.time()
        a, b, c = act.coefficientVectors if isinstance(act, PolyActivation) else (None, None, None)
        res = self._fused(m, lambda inputs, *layer: f.ActivationConvDenseLayer(inputs, a, b, c, *layer))
        self.LastSeconds = time.time() - start
        if self.Verbose:
            print("Layer %s (deferred relinearisation) computed in %.4f seconds layer width (%d,%d)"
                  % (type(self).__name__, self.LastSeconds, m.RowCount, m.ColumnCount))
        m.Dispose()
        return res

    def _prepare_bias(self, m):
        if self.biasVectors is None or self.biasVectors[0].Dim != m.RowCount:
            if self.biasVectors:
                for b in self.biasVectors:
                    b.Dispose()
            scale = self.Source.GetOutputScale() * self.WeightsScale
            f = self.Factory
            self.biasVectors = [f.GetPlainVector(np.full(m.RowCount, self._bias_value(k)), EVectorFormat.dense, scale) for k in range(self.maps())]

    def _fused(self, m, call):
        """call(inputs, gather, weights, bias, M, K) over the columns of m: the whole layer in one factory call."""
        self._prepare_bias(m)
        K = len(self.Offsets)
        M = self.maps() * len(self.Corners)
        if getattr(self, "_gather", None) is None:  # the topology is static: index table built once
            self._gather = np.array([self._gather_row(c) for c in self.Corners] * self.maps(), dtype=np.int32)  # k = map*corners + corner
        inputs = [m.GetColumn(i) for i in range(m.ColumnCount)]
        weights = [self.weightWindows[k // len(self.Corners)] for k in range(M)]
        bias = [self.biasVectors[k // len(self.Corners)] for k in range(M)]
        return self.Factory.GetMatrix(call(inputs, self._gather, weights, bias, M, K), EMatrixFormat.ColumnMajor, CopyVectors=False)

    def Apply(self, m):
        f = self.Factory
        env = f.AllocateComputationEnv()
        if self.Weights is None:  # mean pool: sum of the window, scale absorbs 1/len (PoolLayer.cs:124-145)
            outs = []
            for corner in self.Corners:
                agg = None
                for l in self._gather_row(corner):
                    if l < 0:
                        continue
                    el = m.GetColumn(l)
                    nxt = el if agg is None else agg.Add(el, env)
                    if agg is not None and agg is not el and not _is_column(m, agg):
                        agg.Dispose()
                    agg = nxt
                if _is_column(m, agg):
                    agg = f.CopyVector(agg)
                agg.RegisterScale(agg.Scale * len(self.Offsets))
                outs.append(agg)
            return f.GetMatrix(outs, EMatrixFormat.ColumnMajor, CopyVectors=False)
        if self.Fused and hasattr(f, "ConvDenseLayer"):
            return self._fused(m, f.ConvDenseLayer)
        self._prepare_bias(m)
        M = self.maps() * len(self.Corners)
        res, temps = [], []
        for k in range(M):  # the reference's per-output path (PoolLayer.cs:113-121, 214-223)
            mapIndex, cornerIndex = divmod(k, len(self.Corners))
            cols = []
            for l in self._gather_row(self.Corners[cornerIndex]):
                if l < 0:
                    z = np.zeros(m.RowCount)
                    zv = f.GetEncryptedVector(z, EVectorFormat.dense, m.Scale) if m.IsEncrypted else f.GetPlainVector(z, EVectorFormat.dense, m.Scale)
                    temps.append(zv)
                    cols.append(zv)
                else:
                    cols.append(m.GetColumn(l))
            patch = f.GetMatrix(cols, EMatrixFormat.ColumnMajor, CopyVectors=False)
            patch.DataDisposedExternaly = True
            conv = patch.Mul(self.weightWindows[mapIndex], env)
            res.append(conv.Add(self.biasVectors[mapIndex], env))
            conv.Dispose()
        for t in temps:
            t.Dispose()
        return f.GetMatrix(res, EMatrixFormat.ColumnMajor, CopyVectors=False)


def _is_column(m, v):
    return any(v is c for c in getattr(m, "vectors", []) or [])


def _batchable(f, name, ms, columns=None):
    """The factory's batched entry point `name` when it applies to these matrices (one per client): at least two, encrypted column-major
    matrices with the same column count (`columns` when given) and columns of one dimension, scale and block count.  None otherwise
    (the Raw backend, one client, differing shapes): the layer then applies one matrix at a time."""
    batch = getattr(f, name, None)
    if batch is None or len(ms) < 2:
        return None
    ref = ms[0].vectors[0]
    for m in ms:
        if m.Format != EMatrixFormat.ColumnMajor or m.ColumnCount != ms[0].ColumnCount or (columns is not None and m.ColumnCount != columns):
            return None
        for v in m.vectors:
            if not v.IsEncrypted or v.Dim != ref.Dim or v.Scale != ref.Scale or v.Format != ref.Format or v.vec.blocks != ref.vec.blocks:
                return None
    return batch


class LLPoolLayer(_ConvLayerBase):
    """`NeuralNetworks/LLPoolLayer.cs:10-153`: the input matrix is [corners x offsets] (im2col), one column per offset."""

    def __init__(self, **kw):
        self.HotIndices = None
        super().__init__(**kw)

    def Prepare(self):
        if self.layerPrepared:
            return
        self.ce.Prepare()
        self.kernelSize = int(np.prod(self.KernelShape)) + (1 if self.Bias is None else 0)
        if self.Weights is None:
            return
        self.PrepareWeightsWindows()
        if self.HotIndices is None:
            self.HotIndices = np.ones(len(self.Corners))
        scale = self.Source.GetOutputScale() * self.WeightsScale
        self.biasVectors = [self.Factory.GetPlainVector(self.HotIndices * self._bias_value(k), EVectorFormat.dense, scale) for k in range(self.maps())]
        self.layerPrepared = True

    def Apply(self, m):
        f = self.Factory
        env = f.AllocateComputationEnv()
        if self.Weights is None:
            vec = None
            for i in range(m.ColumnCount):
                c = m.GetColumn(i)
                vec = c if vec is None else vec.Add(c, env)
            vec.RegisterScale(vec.Scale * m.ColumnCount)
            return f.GetMatrix([vec], EMatrixFormat.ColumnMajor, CopyVectors=False)
        res = []
        for k in range(len(self.biasVectors)):
            mul = m.Mul(self.weightWindows[k], env)
            res.append(mul.Add(self.biasVectors[k], env))
            mul.Dispose()
        return f.GetMatrix(res, EMatrixFormat.ColumnMajor, CopyVectors=False)

    def ApplyBatch(self, ms):
        """Every client's convolution in one scalar-MAC call (the MAC is key-independent; each output reads one client's columns), then
        each output's bias."""
        f = self.Factory
        batch = getattr(f, "ConvBatch", None)
        if (batch is None or len(ms) < 2 or self.Weights is None or any(m.Format != EMatrixFormat.ColumnMajor or not m.IsEncrypted for m in ms)
                or any(m.ColumnCount != ms[0].ColumnCount or m.vectors[0].Dim != ms[0].vectors[0].Dim for m in ms)):
            return super().ApplyBatch(ms)
        env = f.AllocateComputationEnv()
        out = []
        for muls in batch(ms, self.weightWindows):
            res = [mul.Add(self.biasVectors[k], env) for k, mul in enumerate(muls)]
            for mul in muls:
                mul.Dispose()
            out.append(f.GetMatrix(res, EMatrixFormat.ColumnMajor, CopyVectors=False))
        return out


class LLVectorizeLayer(BaseLayer):
    """`NeuralNetworks/LLVectorizeLayer.cs:8-24`"""

    OutputDim = -1

    def Apply(self, m):
        vec = m.ConvertToColumnVector(self.Factory.AllocateComputationEnv())
        return self.Factory.GetMatrix([vec], EMatrixFormat.ColumnMajor, CopyVectors=False)

    def ApplyBatch(self, ms):
        """Every client's vectorisation in one pass: the rotations of all clients share key-switch waves (cnhe_vecs_stack_batch)."""
        f = self.Factory
        batch = getattr(f, "StackBatch", None)
        if batch is None or len(ms) < 2 or any(m.ColumnCount != ms[0].ColumnCount for m in ms):
            return super().ApplyBatch(ms)
        return [f.GetMatrix([v], EMatrixFormat.ColumnMajor, CopyVectors=False) for v in batch(ms)]

    def OutputDimension(self):
        return self.OutputDim if self.OutputDim > 0 else super().OutputDimension()


class LLDenseLayer(BaseLayer):
    """`NeuralNetworks/LLDenseLayer.cs:10-76`: row-major plain weights x one encrypted column vector (rotate-and-sum)."""

    def __init__(self, **kw):
        self.Weights = None
        self.Bias = None
        self.WeightsScale = 1.0
        self.InputFormat = EVectorFormat.dense
        self.ForceDenseFormat = False
        self.WeightsMatrix = None
        self.BiasVector = None
        self.Shard = None  # (rank, world, process group): split the rows of this layer over the ranks of ONE inference (SURVEY.md 8e)
        # "rows": the reference's product (per row a multiply, SumAllSlots and a one-hot mask); "diagonal": the baby-step / giant-step
        # diagonal product (DESIGN.md section 4.10), same decrypted output, ForceDenseFormat with a dense input only, no Shard.  The Raw
        # backend computes M v directly either way.  "folded": the folded diagonal product for layers with few rows (DESIGN.md section
        # 4.10, cnhe_diag_prepare_folded), a dense input with or without ForceDenseFormat, no Shard; its output is always dense of dim
        # len(Bias), and so is the Raw backend's.
        self.Method = "rows"
        self.DiagonalMatrix = None
        # "diagonal" and "folded" only: device bytes the prepared matrix may spend on holding giant-step groups of its diagonals in NTT form, so that
        # each product skips their lift and forward transforms (bit-identical outputs); 0 holds none, None the whole matrix.  The Raw
        # backend ignores it.
        self.DiagonalNttBytes = 0
        self._first_row = 0
        super().__init__(**kw)

    def GetOutputScale(self):
        return self.WeightsScale * self.Source.GetOutputScale()

    def Prepare(self):
        if self.layerPrepared:
            return
        if self.ForceDenseFormat and self.InputFormat == EVectorFormat.sparse:
            raise Exception("forcing dense format is only available when the input is dense")
        if self.Method not in ("rows", "diagonal", "folded"):
            raise Exception("unknown dense layer method %r" % (self.Method,))
        if self.Method == "diagonal" and not (self.ForceDenseFormat and self.InputFormat == EVectorFormat.dense):
            raise Exception("the diagonal method needs ForceDenseFormat and a dense input")
        if self.Method == "folded" and self.InputFormat != EVectorFormat.dense:
            raise Exception("the folded method needs a dense input")
        if self.Method != "rows" and self.Shard is not None:
            raise Exception("the %s method cannot be combined with Shard" % self.Method)
        if self.DiagonalNttBytes != 0 and self.Method == "rows":
            raise Exception("DiagonalNttBytes needs the diagonal or the folded method")
        if self.DiagonalNttBytes is not None and not 0 <= self.DiagonalNttBytes < 1 << 64:
            raise Exception("DiagonalNttBytes must be None or a byte count in [0, 2**64)")
        f = self.Factory
        rows = len(self.Bias)
        w = np.asarray(self.Weights, dtype=np.float64).reshape(rows, -1)
        bscale = self.Source.GetOutputScale() * self.WeightsScale
        if self.Shard is not None and self.InputFormat == EVectorFormat.dense and not isinstance(f, RawFactory):
            from .parallel import row_slice
            self._first_row, count = row_slice(rows, self.Shard[0], self.Shard[1])
            w = w[self._first_row:self._first_row + count]  # this rank encodes and holds its slice of the rows only
        else:
            self.Shard = None
        if self.InputFormat == EVectorFormat.dense:
            self.BiasVector = f.GetPlainVector(np.asarray(self.Bias), EVectorFormat.dense if self._dense_out() else EVectorFormat.sparse, bscale)
            self.WeightsMatrix = f.GetPlainMatrix(w, EMatrixFormat.RowMajor, self.WeightsScale)
        else:
            self.BiasVector = f.GetPlainVector(np.asarray(self.Bias), EVectorFormat.dense, bscale)
            self.WeightsMatrix = f.GetPlainMatrix(w, EMatrixFormat.ColumnMajor, self.WeightsScale)
        if self.Method != "rows" and hasattr(self.WeightsMatrix, "PrepareDiagonal"):
            fold = 0 if self.Method == "folded" else None
            self.DiagonalMatrix = self.WeightsMatrix.PrepareDiagonal(ntt_bytes=self.DiagonalNttBytes, fold_width=fold)
            self.WeightsMatrix.Dispose()  # the diagonals replace the row plaintexts
            self.WeightsMatrix = None
        self.layerPrepared = True

    def OutputDimension(self):
        return len(self.Bias)

    def _dense_out(self):
        return self.ForceDenseFormat or self.Method == "folded"

    def Apply(self, m):
        if m.ColumnCount > 1:
            raise Exception("Expecting only one column")
        env = self.Factory.AllocateComputationEnv()
        if self.DiagonalMatrix is not None:
            mul = self.Factory.MulDiagonalBatch(self.DiagonalMatrix, [m.GetColumn(0)])[0]
        elif self.Shard is not None:
            from . import parallel
            rank, world, group = self.Shard
            rows = len(self.Bias)
            part = self.WeightsMatrix.MulRows(m.GetColumn(0), self.ForceDenseFormat, self._first_row, rows)
            if self.ForceDenseFormat:  # partial sums at their global columns: all-gather + local modular adds
                mul = parallel.allreduce_ciphertext_sum(self.Factory, part, group)
            else:                      # this rank's sparse elements: concatenate the slices
                mul = parallel.allgather_sparse_elements(self.Factory, part, [parallel.row_slice(rows, r, world)[1] for r in range(world)], group)
            if mul is not part:
                part.Dispose()
        else:
            mul = self.WeightsMatrix.Mul(m.GetColumn(0), env, self._dense_out())
        res = mul.Add(self.BiasVector, env)
        mul.Dispose()
        return self.Factory.GetMatrix([res], EMatrixFormat.ColumnMajor, CopyVectors=False)

    def ApplyBatch(self, ms):
        """Every client's row-major product in one pass (cnhe_mat_mul_rowmajor_batch), then each one's bias."""
        f = self.Factory
        if self.DiagonalMatrix is not None:  # every client's diagonal product in one pass
            env = f.AllocateComputationEnv()
            out = []
            for mul in f.MulDiagonalBatch(self.DiagonalMatrix, [self._single_column(m) for m in ms]):
                out.append(f.GetMatrix([mul.Add(self.BiasVector, env)], EMatrixFormat.ColumnMajor, CopyVectors=False))
                mul.Dispose()
            return out
        batch = getattr(f, "MulRowMajorBatch", None)
        if (batch is None or len(ms) < 2 or self.Shard is not None or self.InputFormat != EVectorFormat.dense or not self.WeightsMatrix.Batched
                or any(m.ColumnCount != 1 or not m.GetColumn(0).IsEncrypted or m.GetColumn(0).vec.blocks != 1 for m in ms)):
            return super().ApplyBatch(ms)
        env = f.AllocateComputationEnv()
        out = []
        for mul in batch(self.WeightsMatrix, [m.GetColumn(0) for m in ms], self._dense_out()):
            out.append(f.GetMatrix([mul.Add(self.BiasVector, env)], EMatrixFormat.ColumnMajor, CopyVectors=False))
            mul.Dispose()
        return out

    @staticmethod
    def _single_column(m):
        if m.ColumnCount > 1:
            raise Exception("Expecting only one column")
        return m.GetColumn(0)

    def Dispose(self):
        if self.WeightsMatrix is not None:
            self.WeightsMatrix.Dispose()
        if self.DiagonalMatrix is not None:
            self.DiagonalMatrix.Dispose()
        if self.BiasVector is not None:
            self.BiasVector.Dispose()
        self.WeightsMatrix = self.DiagonalMatrix = self.BiasVector = None


class LLSingleLineReader(MatrixSource):
    """One image per GetNext() as a single column vector (`LLSingleLineReader.cs`; TSV parsing replaced by an in-memory array)."""

    def __init__(self, features, Scale, NormalizationFactor):
        super().__init__(features, Scale, NormalizationFactor, MaxSlots=1)

    def GetNext(self):
        if self.pos >= len(self.features):
            self.pos = 0
        f = self.features[self.pos] * self.NormalizationFactor
        self.pos += 1
        return RawMatrix(f.reshape(-1, 1), self.Scale, EMatrixFormat.ColumnMajor, 0)


class LLDuplicateLayer(BaseLayer):
    """`NeuralNetworks/LLDuplicateLayer.cs:8-29`: every column is replicated `Count` times at power-of-two strides."""

    Count = 1

    def Apply(self, m):
        env = self.Factory.AllocateComputationEnv()
        cols = [m.GetColumn(i).Duplicate(int(self.Count), env) for i in range(m.ColumnCount)]
        return self.Factory.GetMatrix(cols, m.Format, CopyVectors=False)

    def ApplyBatch(self, ms):
        """Every column of every client duplicated in one pass (cnhe_vecs_duplicate_batch)."""
        f = self.Factory
        batch = _batchable(f, "DuplicateBatch", ms)
        if batch is None:
            return super().ApplyBatch(ms)
        n = ms[0].ColumnCount
        out = batch([v for m in ms for v in m.vectors], int(self.Count))
        return [f.GetMatrix(out[b * n:(b + 1) * n], m.Format, CopyVectors=False) for b, m in enumerate(ms)]

    def OutputDimension(self):
        shift, dim = 1, self.Source.OutputDimension()
        while shift < dim:
            shift *= 2
        return shift * int(self.Count)


class LLInterleaveLayer(BaseLayer):
    """`NeuralNetworks/LLInterleaveLayer.cs:12-56`: keep the selected slots of every column (mask), then pack the columns into one
    vector, column c shifted by c*Shift slots."""

    def __init__(self, **kw):
        self.Shift = 0
        self.SelectedIndices = None
        self.InputGrossDimension = -1
        self.mask = None
        super().__init__(**kw)

    def Prepare(self):
        if self.mask is not None:
            return
        if self.InputGrossDimension < 0:
            self.InputGrossDimension = max(self.SelectedIndices) + 1
        hot = np.zeros(self.InputGrossDimension)
        hot[list(self.SelectedIndices)] = 1.0
        self.mask = self.Factory.GetPlainVector(hot, EVectorFormat.dense, 1)

    def Apply(self, m):
        f = self.Factory
        env = f.AllocateComputationEnv()
        clean = [m.GetColumn(i).PointwiseMultiply(self.mask, env) for i in range(m.ColumnCount)]
        cm = f.GetMatrix(clean, EMatrixFormat.ColumnMajor, CopyVectors=False)
        packed = cm.Interleave(self.Shift, env)
        cm.Dispose()
        return f.GetMatrix([packed], EMatrixFormat.ColumnMajor, CopyVectors=False)

    def ApplyBatch(self, ms):
        """Every client's mask products in one pass (cnhe_vecs_multiply_plain), then every client's interleave (cnhe_vecs_interleave_batch)."""
        f = self.Factory
        if _batchable(f, "MultiplyPlainBatch", ms) is None or not hasattr(f, "InterleaveBatch"):
            return super().ApplyBatch(ms)
        n = ms[0].ColumnCount
        clean = f.MultiplyPlainBatch([v for m in ms for v in m.vectors], self.mask)
        cms = [f.GetMatrix(clean[b * n:(b + 1) * n], EMatrixFormat.ColumnMajor, CopyVectors=False) for b in range(len(ms))]
        packed = f.InterleaveBatch(cms, self.Shift)
        for cm in cms:
            cm.Dispose()
        return [f.GetMatrix([v], EMatrixFormat.ColumnMajor, CopyVectors=False) for v in packed]

    def OutputDimension(self):
        return self.InputGrossDimension

    def Dispose(self):
        if self.mask is not None:
            self.mask.Dispose()
        self.mask = None


class LLPackedDenseLayer(BaseLayer):
    """`NeuralNetworks/LLPackedDenseLayer.cs:10-76`: `PackingCount` weight rows share one plaintext, each in its own
    `PackingShift`-slot segment; one multiply + partial rotate-and-sum evaluates them all against the duplicated input, the
    result of segment c landing in its last slot (where the bias sits)."""

    def __init__(self, **kw):
        self.Weights = None
        self.Bias = None
        self.WeightsScale = 1.0
        self.PackingCount = 1
        self.PackingShift = 0
        self.WeightsMatrix = None
        self.BiasMatrix = None
        super().__init__(**kw)

    def GetOutputScale(self):
        return self.WeightsScale * self.Source.GetOutputScale()

    def Prepare(self):
        if self.layerPrepared:
            return
        maps = len(self.Bias)
        w = np.asarray(self.Weights, dtype=np.float64).reshape(maps, -1)
        pc, ps = int(self.PackingCount), int(self.PackingShift)
        rows = (maps + pc - 1) // pc
        stacked = np.zeros((rows, pc * ps))
        bias = np.zeros((rows, pc * ps))
        for i in range(maps):
            row, col = divmod(i, pc)
            stacked[row, col * ps: col * ps + w.shape[1]] = w[i]
            bias[row, (col + 1) * ps - 1] = self.Bias[i]
        f = self.Factory
        self.BiasMatrix = f.GetPlainMatrix(bias, EMatrixFormat.RowMajor, self.Source.GetOutputScale() * self.WeightsScale)
        self.WeightsMatrix = f.GetPlainMatrix(stacked, EMatrixFormat.RowMajor, self.WeightsScale)
        self.layerPrepared = True

    def OutputDimension(self):
        return len(self.Bias)

    def Apply(self, m):
        if m.ColumnCount > 1:
            raise Exception("Expecting only one column")
        env = self.Factory.AllocateComputationEnv()
        v = m.GetColumn(0)
        res = []
        for k in range(self.WeightsMatrix.RowCount):
            mul = self.WeightsMatrix.GetRow(k).DotProduct(v, env, length=int(self.PackingShift))
            res.append(mul.Add(self.BiasMatrix.GetRow(k), env))
            mul.Dispose()
        return self.Factory.GetMatrix(res, EMatrixFormat.ColumnMajor, CopyVectors=False)

    def ApplyBatch(self, ms):
        """Every row's partial dot product with every client's vector in one pass (cnhe_mat_dot_rows_batch), then each row's bias."""
        f = self.Factory
        batch = _batchable(f, "DotRowsBatch", ms, columns=1)
        if batch is None or ms[0].vectors[0].vec.blocks != 1:
            return super().ApplyBatch(ms)
        env = f.AllocateComputationEnv()
        out = []
        for muls in batch(self.WeightsMatrix, [m.GetColumn(0) for m in ms], int(self.PackingShift)):
            out.append(f.GetMatrix([mul.Add(self.BiasMatrix.GetRow(k), env) for k, mul in enumerate(muls)], EMatrixFormat.ColumnMajor, CopyVectors=False))
            for mul in muls:
                mul.Dispose()
        return out

    def Dispose(self):
        for mat in (self.WeightsMatrix, self.BiasMatrix):
            if mat is not None:
                mat.Dispose()
        self.WeightsMatrix = self.BiasMatrix = None


class LLInterleavedDenseLayer(BaseLayer):
    """`NeuralNetworks/LLInterleavedDenseLayer.cs:12-77`: dense layer whose inputs sit at the slots an LLInterleaveLayer left them in."""

    def __init__(self, **kw):
        self.Weights = None
        self.Bias = None
        self.WeightsScale = 1
        self.Shift = 0
        self.SelectedIndices = None
        self.WeightsMatrix = None
        self.BiasVector = None
        super().__init__(**kw)

    def GetOutputScale(self):
        return self.Source.GetOutputScale() * self.WeightsScale

    def OutputDimension(self):
        return len(self.Bias)

    def _targets(self, count):
        out, offset = [], 0
        while count > 0:
            for s in self.SelectedIndices:
                if count == 0:
                    break
                out.append(s + offset)
                count -= 1
            offset += self.Shift
        return out

    def Prepare(self):
        if self.layerPrepared:
            return
        rows = len(self.Bias)
        small = np.asarray(self.Weights, dtype=np.float64).reshape(rows, -1)
        big = np.zeros((rows, self.Source.OutputDimension()))
        for i, t in enumerate(self._targets(small.shape[1])):
            big[:, t] = small[:, i]
        f = self.Factory
        self.BiasVector = f.GetPlainVector(np.asarray(self.Bias, dtype=np.float64), EVectorFormat.sparse, self.GetOutputScale())
        self.WeightsMatrix = f.GetPlainMatrix(big, EMatrixFormat.RowMajor, self.WeightsScale)
        self.layerPrepared = True

    def Apply(self, m):
        env = self.Factory.AllocateComputationEnv()
        mul = self.WeightsMatrix.Mul(m.GetColumn(0), env)
        v = mul.Add(self.BiasVector, env)
        mul.Dispose()
        return self.Factory.GetMatrix([v], EMatrixFormat.ColumnMajor, CopyVectors=False)

    def ApplyBatch(self, ms):
        """Every client's sparse row-major product in one pass (cnhe_mat_mul_rowmajor_batch), then each one's bias."""
        f = self.Factory
        batch = _batchable(f, "MulRowMajorBatch", ms, columns=1)
        if batch is None or ms[0].vectors[0].vec.blocks != 1 or not self.WeightsMatrix.Batched:
            return super().ApplyBatch(ms)
        env = f.AllocateComputationEnv()
        out = []
        for mul in batch(self.WeightsMatrix, [m.GetColumn(0) for m in ms], False):
            out.append(f.GetMatrix([mul.Add(self.BiasVector, env)], EMatrixFormat.ColumnMajor, CopyVectors=False))
            mul.Dispose()
        return out

    def Dispose(self):
        if self.WeightsMatrix is not None:
            self.WeightsMatrix.Dispose()
        if self.BiasVector is not None:
            self.BiasVector.Dispose()
        self.WeightsMatrix = self.BiasVector = None


class LLPreConvLayer(BaseLayer):
    """`NeuralNetworks/LLPreConvLayer.cs:13-170`: builds the im2col columns of a convolution *homomorphically* from one encrypted
    image vector.  Column i (kernel offset i) is a permutation of the image: for every block of output rows, mask the pixels that
    offset touches and rotate them so that output position `CornersMap[j]` holds corner j's pixel -- the same map for every offset,
    so the following LLPoolLayer is a plain column-wise weighted sum (with `HotIndices` marking the live slots for the bias)."""

    def __init__(self, **kw):
        self.ce = ConvolutionEngine()
        self.UseAxisForBlocks = None
        self.outputDim = -1
        self.shifts = None
        self.masks = None
        self.CornersMap = None
        self._hot = None
        super().__init__(**kw)

    InputShape = property(lambda s: s.ce.InputShape, lambda s, v: setattr(s.ce, "InputShape", list(v)))
    KernelShape = property(lambda s: s.ce.KernelShape, lambda s, v: setattr(s.ce, "KernelShape", list(v)))
    Stride = property(lambda s: s.ce.Stride, lambda s, v: setattr(s.ce, "Stride", list(v)))
    Padding = property(lambda s: s.ce.Padding, lambda s, v: setattr(s.ce, "Padding", list(v)))
    Upperpadding = property(lambda s: s.ce.Upperpadding, lambda s, v: setattr(s.ce, "Upperpadding", list(v)))
    Lowerpadding = property(lambda s: s.ce.Lowerpadding, lambda s, v: setattr(s.ce, "Lowerpadding", list(v)))

    @property
    def HotIndices(self):
        if not self.layerPrepared:
            self.Prepare()
        return self._hot

    def _block_offsets(self):
        """Offsets of the stride cosets used as blocks: an odometer over the flagged axes, axis 0 fastest (:31-59)."""
        n = len(self.Stride)
        step = [1] * n
        for i in range(1, n):
            step[i] = step[i - 1] * self.InputShape[i - 1]
        block, offset, out = [0] * n, 0, []
        while True:
            out.append(offset)
            advanced = False
            for i in range(n):
                if not self.UseAxisForBlocks[i]:
                    continue
                block[i] += 1
                offset += step[i]
                if block[i] < self.Stride[i]:
                    advanced = True
                    break
                offset -= block[i] * step[i]
                block[i] = 0
            if not advanced:
                return out

    def Prepare(self):
        if self.layerPrepared:
            return
        ce = self.ce
        ce.Prepare()
        if self.UseAxisForBlocks is None:
            self.UseAxisForBlocks = [True] * len(self.InputShape)
        dim = int(np.prod(ce.InputShape))
        row = dim // ce.InputShape[0]
        boff = self._block_offsets()
        nb = len(boff)
        first_axis = sorted({c[0] for c in ce.Corners})
        small = len(first_axis) // nb
        large = -(-len(first_axis) // nb)
        n_large = len(first_axis) - nb * small
        cmap = [-1] * len(ce.Corners)
        f = self.Factory
        self.masks, self.shifts = [], []
        for off in ce.Offsets:
            sh = [0] * nb
            for j in range(nb):
                size = small if j > n_large else large  # (sic) `>`: block n_large still counts as large in the shift recurrence (:99)
                sh[j] = ce.Location(None, off, ce.InputShape) if j == 0 else sh[j - 1] + boff[j - 1] - boff[j] + size * ce.Stride[0] * row
            sel = [[] for _ in range(nb)]
            for j, corner in enumerate(ce.Corners):
                loc = ce.Location(corner, off, ce.InputShape)
                cid = (corner[0] - ce.Corners[0][0]) // ce.Stride[0]
                block = cid // large if cid < large * n_large else n_large + (cid - large * n_large) // small
                if loc >= 0:
                    sel[block].append(loc)
                    where = loc - sh[block]
                    if cmap[j] >= 0 and cmap[j] != where:
                        raise Exception("Internal Error")
                    cmap[j] = where
            mk = []
            for s in sel:
                if s:
                    hot = np.zeros(dim)
                    hot[s] = 1.0
                    mk.append(f.GetPlainVector(hot, EVectorFormat.dense, 1))
                else:
                    mk.append(None)
            self.masks.append(mk)
            self.shifts.append(sh)
        large_max = 0 if n_large == 0 else row * (1 + ce.Stride[0] * (large - 1)) + boff[n_large - 1]
        small_max = row * (1 + ce.Stride[0] * (small - 1)) + boff[-1]
        self.outputDim = max(large_max, small_max)
        self.CornersMap = cmap
        self._hot = np.zeros(self.outputDim)
        self._hot[cmap] = 1.0
        self.layerPrepared = True

    def Apply(self, m):
        if m.ColumnCount != 1:
            raise Exception("Expecting only a single column")
        if not self.layerPrepared:
            self.Prepare()
        env = self.Factory.AllocateComputationEnv()
        v = m.GetColumn(0)
        cols = [v.Permute(self.masks[k], self.shifts[k], self.outputDim, env) for k in range(len(self.masks))]
        return self.Factory.GetMatrix(cols, EMatrixFormat.ColumnMajor, CopyVectors=False)

    def ApplyBatch(self, ms):
        """Every client's permutations in one pass (cnhe_vecs_permute_batch): one outer mask product, one wave per rotation hop."""
        f = self.Factory
        batch = _batchable(f, "PermuteBatch", ms, columns=1)
        if batch is None:
            return super().ApplyBatch(ms)
        if not self.layerPrepared:
            self.Prepare()
        return [f.GetMatrix(cols, EMatrixFormat.ColumnMajor, CopyVectors=False)
                for cols in batch([m.GetColumn(0) for m in ms], self.masks, self.shifts, self.outputDim)]

    def OutputDimension(self):
        if not self.layerPrepared:
            self.Prepare()
        return self.outputDim

    def RearrangeWeights(self, weights):
        """Weights of the next dense layer re-indexed from corner order to the slot order this layer produces (:154-168)."""
        if not self.layerPrepared:
            self.Prepare()
        weights = np.asarray(weights, dtype=np.float64)
        nc = len(self.ce.Corners)
        maps = len(weights) // nc
        out = np.zeros(maps * self.outputDim)
        for i in range(maps):
            for j in range(nc):
                out[i * self.outputDim + self.CornersMap[j]] = weights[j + i * nc]
        return out

    def Dispose(self):
        if self.masks:
            for mk in self.masks:
                for v in mk:
                    if v is not None:
                        v.Dispose()
        self.masks = None
