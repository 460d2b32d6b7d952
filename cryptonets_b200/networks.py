"""Network topologies of the reference apps, built from the layer API exactly as the C# mains build them.

cryptonets_mnist  <- `CryptoNets/CryptoNets.cs:12-75`   (config 2 of BASELINE.json)
lola_small        <- `LowLatencyCryptoNets/LoLaCryptonets.cs:280-329` (config 3)
lola / lola_dense / lola_large / lola_cifar <- the other mains of `LoLaCryptonets.cs` and `CifarCryptoNet/LolaCifarCryptoNet.cs` (config 4)
Trained parameters come from cryptonets_b200/models/*.npz (generated from the reference's shipped constants and CSV files by
tools/extract_reference_weights.py) or, when a file is absent, from a seeded generator of the same shapes."""
import os

import numpy as np

from .interfaces import EVectorFormat
from .layers import (ConvolutionEngine, EncryptLayer, LLConvReader, LLDenseLayer, LLDuplicateLayer, LLInterleavedDenseLayer, LLInterleaveLayer,
                     LLPackedDenseLayer, LLPoolLayer, LLPreConvLayer, LLSingleLineReader, LLVectorizeLayer, MatrixSource, PoolLayer,
                     SquareActivation, TimingLayer)

_MODELS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "models")
CRYPTONETS_PRIMES = [549764251649, 549764284417]  # CryptoNets.cs:17
LOLA_SMALL_PRIMES = [2277377, 2424833]            # LoLaCryptonets.cs:285
LOLA_PRIMES = [557057, 638977, 737281, 786433]    # LoLaCryptonets.cs:208 (N=8192, default decomposition bit counts)
LOLA_DENSE_PRIMES = [34359771137, 34360754177]    # LoLaCryptonets.cs:123 (N=16384, w=60, SmallModulusCount=7)
CIFAR_PRIMES = [957181001729, 957181034497]       # LolaCifarCryptoNet.cs:35 (N=16384, w=60, SmallModulusCount=8)
LOLA_LARGE_PRIMES = [2148728833, 2148794369, 2149810177]  # LoLaCryptonets.cs:336 (N=16384, w=60, SmallModulusCount=7)


def load_weights(name, shapes, seed=0):
    path = os.path.join(_MODELS, name)
    if os.path.exists(path):
        z = np.load(path)
        return {k: z[k] for k in z.files}
    rng = np.random.default_rng(seed)
    return {k: rng.normal(0, s, n) for k, (n, s) in shapes.items()}


def cryptonets_weights():
    return load_weights("cryptonets_mnist_weights.npz",
                        dict(Weights_0=(130, 0.4), Weights_1=(84500, 0.006), Weights_3=(1000, 0.1), Biases_2=(100, 0.05), Biases_3=(10, 0.1)))


def lola_small_weights():
    return load_weights("lola_small_weights.npz", dict(Weights_0=(130, 0.4), Weights_1=(8450, 0.05), Biases_1=(10, 0.1)))


def transpose(weights, inputShapeSize, outputMaps):  # CryptoNets.cs:111-122
    res = np.zeros(len(weights))
    for i in range(inputShapeSize):
        for j in range(outputMaps):
            res[i + inputShapeSize * j] = weights[outputMaps * i + j]
    return res


def synthetic_mnist(n_images, seed=20240917):
    """MNIST-shaped synthetic batch (SURVEY 8d): uint8 pixels, ~80% zeros."""
    rng = np.random.default_rng(seed)
    px = rng.integers(0, 256, (n_images, 784))
    px[rng.random((n_images, 784)) < 0.8] = 0
    return px.astype(np.float64)


def cryptonets_mnist(factory, images, batch_size=None, fused=True, weights=None, timing=True, defer_relinearization=False):
    """Returns (network, reader).  network.GetNext() yields the 10-column score matrix of one batch.  defer_relinearization: both dense
    layers square their input and relinearise only their outputs (PoolLayer.DeferRelinearization): same scores, 110 relinearisations per
    plaintext prime instead of 945."""
    w = weights or cryptonets_weights()
    weightscale = 32
    reader = MatrixSource(images, Scale=16.0, NormalizationFactor=1.0 / 256.0, MaxSlots=batch_size or len(images))
    enc = EncryptLayer(Source=reader, Factory=factory)
    src = TimingLayer(Source=enc, StartCounters=["Batch-Time"]) if timing else enc
    conv1 = PoolLayer(Source=src, InputShape=[28, 28], KernelShape=[5, 5], Upperpadding=[1, 1], Stride=[2, 2], MapCount=[5, 1],
                      WeightsScale=weightscale, Weights=w["Weights_0"], Fused=fused)
    act2 = SquareActivation(Source=conv1)
    dense3 = PoolLayer(Source=act2, InputShape=[5 * 13 * 13], KernelShape=[5 * 13 * 13], Stride=[1000], MapCount=[100],
                       Weights=transpose(w["Weights_1"], 5 * 13 * 13, 100), Bias=w["Biases_2"], WeightsScale=weightscale * weightscale, Fused=fused,
                       DeferRelinearization=defer_relinearization)
    act4 = SquareActivation(Source=dense3)
    dense5 = PoolLayer(Source=act4, InputShape=[100], KernelShape=[100], Stride=[1000], MapCount=[10], Weights=w["Weights_3"],
                       Bias=w["Biases_3"], WeightsScale=weightscale, Fused=fused, DeferRelinearization=defer_relinearization)
    net = TimingLayer(Source=dense5, StopCounters=["Batch-Time"]) if timing else dense5
    return net, reader


def lola_small(factory, images, weights=None, dense_method="rows"):
    """dense_method: LLDenseLayer.Method of the 10 x 845 score layer ("rows", the reference's, or "folded": dense scores in one
    ciphertext per plaintext prime)."""
    w = weights or lola_small_weights()
    weightscale = 64
    reader = LLConvReader(images, Scale=16.0, NormalizationFactor=1.0 / 256.0, InputShape=[28, 28], KernelShape=[5, 5], Stride=[2, 2],
                          Upperpadding=[1, 1])
    enc = EncryptLayer(Source=reader, Factory=factory)
    conv1 = LLPoolLayer(Source=enc, InputShape=[28, 28], KernelShape=[5, 5], Upperpadding=[1, 1], Stride=[2, 2], MapCount=[5, 1],
                        WeightsScale=weightscale, Weights=w["Weights_0"])
    vec2 = LLVectorizeLayer(Source=conv1)
    act3 = SquareActivation(Source=vec2)
    dense4 = LLDenseLayer(Source=act3, Bias=w["Biases_1"], Weights=w["Weights_1"], WeightsScale=weightscale, Method=dense_method)
    return dense4, reader


def serve_batch(net, inputs):
    """Runs one inference per client through the layers that follow the network's EncryptLayer, all clients together: each layer takes
    the list of matrices (BaseLayer.ApplyBatch), so the key switches of all clients share waves.  inputs: one encrypted input matrix per
    client, already on the server's factory and bound to that client's key slot (LoadCompactMatrix(..., slot=)); the caller keeps them.
    Returns one output matrix per client -- the same ciphertexts each would get from a server that holds only its keys."""
    chain, layer = [], net
    while not isinstance(layer, EncryptLayer):
        chain.append(layer)
        layer = layer.Source
    chain.reverse()
    for layer in chain:
        if not layer.layerPrepared:
            layer.Prepare()
            layer.layerPrepared = True
    ms = list(inputs)
    for layer in chain:
        out = layer.ApplyBatch(ms)
        for m, o in zip(ms, out):
            if o is not m and not any(m is i for i in inputs):
                m.Dispose()
        ms = out
    return ms


def lola(factory, images, weights=None):
    """LoLa (`LowLatencyCryptoNets/LoLaCryptonets.cs:203-276`): im2col input, 8-way packed dense layer, interleave, square, dense."""
    w = weights or cryptonets_weights()
    weightscale = 32
    reader = LLConvReader(images, Scale=16.0, NormalizationFactor=1.0 / 256.0, InputShape=[28, 28], KernelShape=[5, 5], Stride=[2, 2],
                          Upperpadding=[1, 1])
    enc = EncryptLayer(Source=reader, Factory=factory)
    conv1 = LLPoolLayer(Source=enc, InputShape=[28, 28], KernelShape=[5, 5], Upperpadding=[1, 1], Stride=[2, 2], MapCount=[5, 1],
                        WeightsScale=weightscale, Weights=w["Weights_0"])
    vec2 = LLVectorizeLayer(Source=conv1)
    act3 = SquareActivation(Source=vec2)
    dup4 = LLDuplicateLayer(Source=act3, Count=8)
    dense5 = LLPackedDenseLayer(Source=dup4, Weights=transpose(w["Weights_1"], 5 * 13 * 13, 100), Bias=w["Biases_2"],
                                WeightsScale=weightscale * weightscale, PackingCount=8, PackingShift=1024)
    sel = [1023 + i * 1024 for i in range(8)]
    inter6 = LLInterleaveLayer(Source=dense5, Shift=-1, SelectedIndices=sel)
    act7 = SquareActivation(Source=inter6)
    dense8 = LLInterleavedDenseLayer(Source=act7, Weights=w["Weights_3"], Bias=w["Biases_3"], WeightsScale=weightscale, Shift=-1,
                                     SelectedIndices=sel)
    return dense8, reader


def lola_dense(factory, images, weights=None):
    """LoLa-Dense (`LoLaCryptonets.cs:116-201`): the image arrives as ONE ciphertext; the im2col columns are built homomorphically
    (LLPreConvLayer), 16-way packed dense layer, square, interleave, dense."""
    w = weights or cryptonets_weights()
    weightscale = 32
    reader = LLSingleLineReader(images, Scale=16.0, NormalizationFactor=1.0 / 256.0)
    enc = EncryptLayer(Source=reader, Factory=factory)
    pre1 = LLPreConvLayer(Source=enc, InputShape=[28, 28], KernelShape=[5, 5], Upperpadding=[1, 1], Stride=[2, 2], UseAxisForBlocks=[True, True])
    conv2 = LLPoolLayer(Source=pre1, InputShape=[28, 28], KernelShape=[5, 5], Upperpadding=[1, 1], Stride=[2, 2], MapCount=[5, 1],
                        WeightsScale=weightscale, Weights=w["Weights_0"], HotIndices=pre1.HotIndices)
    vec3 = LLVectorizeLayer(Source=conv2)
    act4 = SquareActivation(Source=vec3)
    dup5 = LLDuplicateLayer(Source=act4, Count=16)
    dense6 = LLPackedDenseLayer(Source=dup5, Weights=pre1.RearrangeWeights(transpose(w["Weights_1"], 5 * 13 * 13, 100)), Bias=w["Biases_2"],
                                WeightsScale=weightscale * weightscale, PackingCount=16, PackingShift=1024)
    act7 = SquareActivation(Source=dense6)
    sel = [1023 + i * 1024 for i in range(16)]
    inter8 = LLInterleaveLayer(Source=act7, Shift=-1, SelectedIndices=sel)
    dense9 = LLInterleavedDenseLayer(Source=inter8, Weights=w["Weights_3"], Bias=w["Biases_3"], WeightsScale=weightscale, Shift=-1,
                                     SelectedIndices=sel)
    return dense9, reader


def cifar_weights(seed=7, synthetic=False):
    """The shipped `CifarWeight.csv` / `CifarBias.csv` (models/lola_cifar_weights.npz): conv 83 x (3*8*8), conv-as-dense 112 x (83*10*10),
    dense 10 x 5488.  synthetic=True (or a missing file): seeded weights with the same shapes and per-layer spread."""
    path = os.path.join(_MODELS, "lola_cifar_weights.npz")
    if not synthetic and os.path.exists(path):
        z = np.load(path)
        return {k: z[k].astype(np.float64) for k in z.files}
    rng = np.random.default_rng(seed)

    def draw(n, std, cap):
        return np.clip(rng.normal(0, std, n), -cap, cap)

    return dict(Weights_0=draw(83 * 192, 0.073, 0.51), Biases_0=draw(83, 0.12, 0.39), Weights_1=draw(112 * 8300, 0.020, 0.11),
                Biases_1=draw(112, 0.12, 0.22), Weights_2=draw(10 * 5488, 0.187, 1.03), Biases_2=draw(10, 0.67, 1.44))


def synthetic_cifar(n_images, seed=20240917):
    return np.random.default_rng(seed).integers(0, 256, (n_images, 3 * 32 * 32)).astype(np.float64)


def lola_cifar(factory, images, weights=None, shard=None, dense_method="rows", diag_ntt_bytes=0, score_method="rows"):
    """LoLa-CIFAR (`CifarCryptoNet/LolaCifarCryptoNet.cs:27-131`): 3x32x32 image as an im2col matrix [196 x 192], conv 83 maps,
    square, the second convolution as a 5488 x 16268 row-major dense layer (rotate-and-sum per row), square, dense 5488 -> 10.
    dense_method: LLDenseLayer.Method of that layer ("rows", the reference's, or "diagonal"); diag_ntt_bytes: its DiagonalNttBytes;
    score_method: the Method of the score layer ("rows" or "folded")."""
    w = weights or cifar_weights()
    reader = LLConvReader(images, Scale=8.0, NormalizationFactor=1.0 / 256.0, InputShape=[3, 32, 32], KernelShape=[3, 8, 8], Stride=[1000, 2, 2],
                          Upperpadding=[0, 1, 1], Lowerpadding=[0, 1, 1])
    enc = EncryptLayer(Source=reader, Factory=factory)
    conv1 = LLPoolLayer(Source=enc, InputShape=[3, 32, 32], KernelShape=[3, 8, 8], Upperpadding=[0, 1, 1], Lowerpadding=[0, 1, 1],
                        Stride=[1000, 2, 2], MapCount=[83, 1, 1], WeightsScale=256.0, Weights=w["Weights_0"], Bias=w["Biases_0"])
    vec2 = LLVectorizeLayer(Source=conv1)
    act3 = SquareActivation(Source=vec2)
    ce = ConvolutionEngine()
    ce.InputShape, ce.KernelShape, ce.Stride, ce.MapCount = [83, 14, 14], [83, 10, 10], [83, 2, 2], [112, 1, 1]
    ce.Upperpadding, ce.Lowerpadding = [0, 4, 4], [0, 4, 4]
    # shard = (rank, world, process group): the 5488 rows of the big dense layer are split over the ranks of ONE inference (SURVEY.md 8e);
    # every rank holds the same keys and input ciphertexts, the partial products are summed through cryptonets_b200/parallel.py
    dense4 = LLDenseLayer(Source=act3, WeightsScale=512.0, Weights=ce.GetDenseWeights(w["Weights_1"]), Bias=ce.GetDenseBias(w["Biases_1"]),
                          InputFormat=EVectorFormat.dense, ForceDenseFormat=True, Shard=shard, Method=dense_method,
                          DiagonalNttBytes=diag_ntt_bytes)
    act5 = SquareActivation(Source=dense4)
    dense6 = LLDenseLayer(Source=act5, Weights=w["Weights_2"], Bias=w["Biases_2"], WeightsScale=512.0, InputFormat=EVectorFormat.dense,
                          Method=score_method)
    return dense6, reader


def lola_large_weights(seed=9, synthetic=False):
    """The shipped `MnistLargeWeight.csv` / `MnistLargeBias.csv` (models/lola_large_weights.npz): conv 83 x (8*8), conv-as-dense
    163 x (83*6*6), dense 10 x 2608.  synthetic=True (or a missing file): seeded weights with the same shapes and spread."""
    path = os.path.join(_MODELS, "lola_large_weights.npz")
    if not synthetic and os.path.exists(path):
        z = np.load(path)
        return {k: z[k].astype(np.float64) for k in z.files}
    rng = np.random.default_rng(seed)

    def draw(n, std, cap):
        return np.clip(rng.normal(0, std, n), -cap, cap)

    return dict(Weights_0=draw(83 * 64, 0.062, 0.46), Biases_0=draw(83, 0.088, 0.35), Weights_1=draw(163 * 83 * 36, 0.025, 0.117),
                Biases_1=draw(163, 0.039, 0.09), Weights_2=draw(10 * 2608, 0.42, 1.63), Biases_2=draw(10, 1.6, 3.9))


def lola_large(factory, images, weights=None, dense_method="rows", diag_ntt_bytes=0, score_method="rows"):
    """Large LoLa (`LoLaCryptonets.cs:330-409`): 28x28 image as im2col [144 x 64], conv 83 maps of 8x8 stride 2 (pixels are NOT
    normalised; the weights carry the 1/256), square, the second convolution (163 maps of 83x6x6, stride 2 over 83x12x12) as a
    2608 x 11952 row-major dense layer with ForceDenseFormat, square, dense 2608 -> 10.  dense_method: that layer's LLDenseLayer.Method,
    diag_ntt_bytes its DiagonalNttBytes; score_method: the Method of the score layer ("rows" or "folded")."""
    w = weights or lola_large_weights()
    reader = LLConvReader(images, Scale=16.0, NormalizationFactor=1.0, InputShape=[1, 28, 28], KernelShape=[1, 8, 8], Stride=[1000, 2, 2],
                          Upperpadding=[0, 1, 1], Lowerpadding=[0, 1, 1])
    enc = EncryptLayer(Source=reader, Factory=factory)
    conv1 = LLPoolLayer(Source=enc, InputShape=[1, 28, 28], KernelShape=[1, 8, 8], Upperpadding=[0, 1, 1], Lowerpadding=[0, 1, 1],
                        Stride=[1000, 2, 2], MapCount=[83, 1, 1], WeightsScale=4096, Weights=np.asarray(w["Weights_0"]) / 256.0, Bias=w["Biases_0"])
    vec2 = LLVectorizeLayer(Source=conv1)
    act3 = SquareActivation(Source=vec2)
    ce = ConvolutionEngine()
    ce.InputShape, ce.KernelShape, ce.Stride, ce.MapCount = [83, 12, 12], [83, 6, 6], [83, 2, 2], [163, 1, 1]
    ce.Padding = [False, False, False]
    dense4 = LLDenseLayer(Source=act3, WeightsScale=64, Weights=ce.GetDenseWeights(w["Weights_1"]), Bias=ce.GetDenseBias(w["Biases_1"]),
                          InputFormat=EVectorFormat.dense, ForceDenseFormat=True, Method=dense_method,
                          DiagonalNttBytes=diag_ntt_bytes)
    act5 = SquareActivation(Source=dense4)
    dense6 = LLDenseLayer(Source=act5, Weights=w["Weights_2"], Bias=w["Biases_2"], WeightsScale=512, InputFormat=EVectorFormat.dense,
                          Method=score_method)
    return dense6, reader
