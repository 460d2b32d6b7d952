"""End-to-end parity of the reference networks on the GPU backend.

(i)  decrypted scores == the Raw (plaintext) backend exactly -- what the reference itself pins (SURVEY 8c);
(ii) ciphertexts of sampled layer outputs == the CPU oracle run on the same input ciphertexts and keys, bit for bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cryptonets():
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import CRYPTONETS_PRIMES
    f = B200BfvFactory(CRYPTONETS_PRIMES, 8192, seed=77)  # CryptoNets.cs:17
    yield f
    f.Dispose()


def test_cryptonets_mnist_scores_equal_raw_backend(cryptonets):
    from cryptonets_b200.networks import cryptonets_mnist, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    imgs = synthetic_mnist(8192, seed=3)
    net, _ = cryptonets_mnist(cryptonets, imgs)
    net.PrepareNetwork()
    scores = net.GetNext().Decrypt()
    raw_net, _ = cryptonets_mnist(RawFactory(8192), imgs, timing=False)
    raw_net.PrepareNetwork()
    want = raw_net.GetNext().Decrypt()
    assert scores.shape == (8192, 10)
    # the encrypted path is exact: compare with exact integer arithmetic on the first 48 images
    exact = _exact_cryptonets(imgs[:48])
    assert np.array_equal(scores[:48], exact)
    # the Raw backend works in doubles while the integers here need ~80 bits and cancel heavily, so it is only good to
    # ~2^-45 of the largest intermediate; it still has to agree on every prediction
    assert np.allclose(scores, want, rtol=1e-9, atol=1e-9 * np.abs(want).max())
    assert np.array_equal(np.argmax(scores, axis=1), np.argmax(want, axis=1))
    assert len(set(np.argmax(scores, axis=1))) > 1


def _exact_cryptonets(images):
    """CryptoNets-MNIST in exact integer arithmetic (Python ints); returns scores as doubles = int / 2^61."""
    from cryptonets_b200.layers import ConvolutionEngine
    from cryptonets_b200.networks import cryptonets_weights, transpose
    w = cryptonets_weights()
    x = np.rint(images / 256.0 * 16.0).astype(np.int64).astype(object)
    ce = ConvolutionEngine()
    ce.InputShape, ce.KernelShape, ce.Stride, ce.Upperpadding, ce.MapCount = [28, 28], [5, 5], [2, 2], [1, 1], [5, 1]
    ce.Prepare()
    w0 = [int(v) for v in np.rint(w["Weights_0"] * 32)]
    n = len(x)
    conv = np.zeros((n, 845), dtype=object)
    for m in range(5):
        bias = int(np.rint(w["Weights_0"][(m + 1) * 26 - 1] * 16.0 * 32))
        for ci, c in enumerate(ce.Corners):
            acc = np.full(n, bias, dtype=object)
            for o in ce.Offsets:
                l = ce.Location(c, o, ce.InputShape)
                if l >= 0:
                    acc = acc + w0[m * 26 + ce.Location(None, o, ce.KernelShape)] * x[:, l]
            conv[:, m * 169 + ci] = acc
    a = conv * conv
    s = (16 * 32) ** 2
    w1 = np.rint(transpose(w["Weights_1"], 845, 100) * 1024).astype(np.int64).astype(object).reshape(100, 845)
    b1 = np.array([int(v) for v in np.rint(w["Biases_2"] * s * 1024)], dtype=object)
    d = a.dot(w1.T) + b1
    a2 = d * d
    s2 = (s * 1024) ** 2
    w3 = np.rint(w["Weights_3"] * 32).astype(np.int64).astype(object).reshape(10, 100)
    b3 = np.array([int(v) for v in np.rint(w["Biases_3"] * float(s2) * 32)], dtype=object)
    out = a2.dot(w3.T) + b3
    return np.array([[float(int(v)) / float(s2 * 32) for v in row] for row in out])


def test_cryptonets_layers_bit_identical_to_oracle(cryptonets):
    from cryptonets_b200.layers import ConvolutionEngine
    from cryptonets_b200.networks import cryptonets_mnist, synthetic_mnist
    from oracle.oracle_py import Oracle
    f = cryptonets
    imgs = synthetic_mnist(8192, seed=4)
    net, reader = cryptonets_mnist(f, imgs, timing=False)
    net.PrepareNetwork()
    # walk the chain by hand to keep the intermediate matrices
    dense5 = net
    act4 = dense5.Source
    dense3 = act4.Source
    act2 = dense3.Source
    conv1 = act2.Source
    enc = conv1.Source
    x = enc.Apply(reader.GetNext())
    c1 = conv1.Apply(x)
    a2 = act2.Apply(c1)
    d3 = dense3.Apply(a2)
    for ch, t in enumerate(f.engine.primes):
        orc = Oracle(t, 8192, -1, 10, 20)
        orc.keygen(77 + ch)
        assert np.array_equal(f.engine.export_key(ch, 2), orc.relin_keys().ravel())
        # conv layer, three sampled outputs (first, middle, last)
        ce = conv1.ce
        for m in (0, 400, 844):
            mapIndex, corner = divmod(m, 169)
            rows = [ce.Location(ce.Corners[corner], o, ce.InputShape) for o in ce.Offsets]
            used = sorted(set(r for r in rows if r >= 0))
            cts = np.stack([x.GetColumn(i).vec.export_raw(ch, 0) for i in used])
            gather = np.array([[used.index(r) if r >= 0 else -1 for r in rows]], dtype=np.int32)
            w = np.rint(np.array([conv1._weight(o, mapIndex * 26) for o in ce.Offsets]) * 32)
            wres = np.where(w < 0, w + t, w).astype(np.uint64)
            b = np.rint(conv1._bias_value(mapIndex) * 16.0 * 32)
            bres = np.array([b + t if b < 0 else b]).astype(np.uint64)
            want = orc.mac_layer(cts, gather, wres, bres, 1, 25)
            assert np.array_equal(c1.GetColumn(m).vec.export_raw(ch, 0), want), (ch, m)
        # square activation, sampled
        for m in (0, 511, 844):
            src = c1.GetColumn(m).vec.export_raw(ch, 0)
            want = orc.square_layer(src)
            assert np.array_equal(a2.GetColumn(m).vec.export_raw(ch, 0), want), (ch, m)
        # dense 845 -> 100, one sampled output over all 845 inputs
        cts = np.stack([a2.GetColumn(i).vec.export_raw(ch, 0) for i in range(845)])
        m = 37
        w = np.rint(dense3.Weights[m * 845:(m + 1) * 845] * 1024)
        wres = np.where(w < 0, w + t, w).astype(np.uint64)
        b = np.rint(dense3.Bias[m] * (16.0 * 32) ** 2 * 1024)
        big = f.bigFactor
        bres = np.array([int(b) % big % t], dtype=np.uint64)
        want = orc.mac_layer(cts, None, wres, bres, 1, 845, threads=8)
        assert np.array_equal(d3.GetColumn(m).vec.export_raw(ch, 0), want), ch


def test_cryptonets_unfused_path_matches_fused(cryptonets):
    """PoolLayer with Fused=False replays the reference's per-output Mul/Add sequence (fresh zero encryptions on padded taps);
    decrypted results must agree with the fused layer call."""
    from cryptonets_b200.layers import EncryptLayer, MatrixSource, PoolLayer
    from cryptonets_b200.networks import cryptonets_weights, synthetic_mnist
    imgs = synthetic_mnist(8192, seed=5)
    outs = []
    for fused in (True, False):
        reader = MatrixSource(imgs, Scale=16.0, NormalizationFactor=1 / 256.0)
        enc = EncryptLayer(Source=reader, Factory=cryptonets)
        conv = PoolLayer(Source=enc, InputShape=[28, 28], KernelShape=[5, 5], Upperpadding=[1, 1], Stride=[2, 2], MapCount=[1, 1],
                         WeightsScale=32, Weights=cryptonets_weights()["Weights_0"][:26], Fused=fused)
        conv.PrepareNetwork()
        outs.append(conv.GetNext().Decrypt())
    assert np.array_equal(outs[0], outs[1])


def _last_layer_needs(factory, N, mtilde_centered=0):
    """Bits the last LLDenseLayer consumes by the analytic noise model (tools/noise_model.py, validated per operation against the measured
    trace in profiles/r02_noise_trace.md): one dense multiply_plain, log2((t/sqrt12) sqrt N), plus the root-sum-square growth of the
    rotate-and-sum over the N slots, 0.5 log2 N."""
    import importlib.util
    import math
    import os
    spec = importlib.util.spec_from_file_location("noise_model", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "noise_model.py"))
    nm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(nm)
    eng = factory.engine
    rec = dict(N=N, q=eng.q, primes=eng.primes, mtilde_centered=mtilde_centered, dbc=10, dbc_galois=20)
    return nm.Model(rec, 0).plain_gain() + 0.5 * math.log2(N)


def _layer_chain(net):
    out, p = [], net
    while p is not None and hasattr(p, "Source"):
        out.append(p)
        p = p.Source
    return out[::-1]


@pytest.mark.parametrize("small_modulus_count", [4, 3])
def test_lola_small_scores_equal_raw_backend(small_modulus_count):
    """LoLa-small topology (LoLaCryptonets.cs:280-329).  With the reference's SmallModulusCount=3 (130-bit q) the invariant noise budget
    is spent before the last layer finishes -- 55 bits left after the w=40 rotations of LLVectorizeLayer, ~20 after the square, and the
    845-slot MultiplyPlain of LLDenseLayer costs ~27 -- in any faithful BFV (our ciphertexts are bit-identical to the SEAL-3.2 oracle),
    so with k=3 the layers are compared up to the square activation and the budget is reported; with one more prime (k=4) the whole
    network must equal the Raw backend exactly."""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import LOLA_SMALL_PRIMES, lola_small, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    f = B200BfvFactory(LOLA_SMALL_PRIMES, 8192, DecompositionBitCount=40, GaloisDecompositionBitCount=40,
                       SmallModulusCount=small_modulus_count, seed=5)
    try:
        imgs = synthetic_mnist(2, seed=6)
        net, rd = lola_small(f, imgs)
        net.PrepareNetwork()
        raw_net, rrd = lola_small(RawFactory(8192), imgs)
        raw_net.PrepareNetwork()
        if small_modulus_count == 4:
            for batched in (True, False):
                net.WeightsMatrix.Batched = batched
                got = net.GetNext().Decrypt().reshape(-1)
                want = raw_net.GetNext().Decrypt().reshape(-1)
                assert np.array_equal(got, want)
        else:
            ma, mb = rd.GetNext(), rrd.GetNext()
            for A, B in list(zip(_layer_chain(net), _layer_chain(raw_net)))[1:-1]:
                ma, mb = A.Apply(ma), B.Apply(mb)
                assert np.array_equal(np.asarray(ma.Decrypt()), np.asarray(mb.Decrypt())), type(A).__name__
            budget = min(f.engine.noise_budget(v.vec, ch, 0) for v in ma.vectors for ch in range(2))
            # what is left for the dense layer is less than its multiply_plain + rotate-and-sum consume: k=3 cannot decrypt the scores
            assert 0 < budget < _last_layer_needs(f, 8192)
    finally:
        f.Dispose()


def _compare_layerwise(net, raw_net, rd, rrd, upto=None):
    """Apply the two layer chains side by side; returns the last pair of matrices.  Layers whose output carries unselected slots
    (packed dense: partial sums outside the segment ends) are compared only through the layers that consume them."""
    ma, mb = rd.GetNext(), rrd.GetNext()
    pairs = list(zip(_layer_chain(net), _layer_chain(raw_net)))[1:]  # [0] is the reader
    for A, B in pairs[:upto]:
        ma, mb = A.Apply(ma), B.Apply(mb)
    return ma, mb


def test_lola_scores_equal_raw_backend():
    """LoLa (LoLaCryptonets.cs:203-276; 4 plaintext primes, N=8192, default moduli and decomposition): LLPoolLayer, LLVectorizeLayer,
    square, LLDuplicateLayer, LLPackedDenseLayer, LLInterleaveLayer, square, LLInterleavedDenseLayer on one encrypted image."""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import LOLA_PRIMES, lola, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    f = B200BfvFactory(LOLA_PRIMES, 8192, seed=5)
    try:
        imgs = synthetic_mnist(2, seed=6)
        net, _ = lola(f, imgs)
        net.PrepareNetwork()
        raw_net, _ = lola(RawFactory(8192), imgs)
        raw_net.PrepareNetwork()
        for _ in range(2):
            out = net.GetNext()
            budget = min(f.engine.noise_budget(v.vec, ch, 0) for v in out.vectors for ch in range(f.engine.P))
            got = np.asarray(out.Decrypt()).reshape(-1)
            want = np.asarray(raw_net.GetNext().Decrypt()).reshape(-1)
            assert budget > 0
            assert np.allclose(got, want, rtol=1e-9, atol=1e-9) and got.argmax() == want.argmax()
    finally:
        f.Dispose()


@pytest.mark.parametrize("small_modulus_count", [8, 7])
def test_lola_dense_scores_equal_raw_backend(small_modulus_count):
    """LoLa-Dense (LoLaCryptonets.cs:116-201; N=16384, w=60): the im2col columns are built homomorphically by LLPreConvLayer.
    With the reference's SmallModulusCount=7 (341-bit q, 35-bit t) a SEAL-3.2-faithful BFV starts at 270 bits of budget (the
    Delta*m rounding term of 3.2's encryption is ~t/2) and the nine plaintext/ciphertext multiplications of the topology need
    ~283: layers are compared through the interleave layer (36 bits left), the last dense layer cannot decrypt.  With one more
    prime the whole network equals the Raw backend."""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import LOLA_DENSE_PRIMES, lola_dense, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    f = B200BfvFactory(LOLA_DENSE_PRIMES, 16384, DecompositionBitCount=60, GaloisDecompositionBitCount=60,
                       SmallModulusCount=small_modulus_count, seed=5)
    try:
        imgs = synthetic_mnist(1, seed=6)
        net, rd = lola_dense(f, imgs)
        net.PrepareNetwork()
        raw_net, rrd = lola_dense(RawFactory(16384), imgs)
        raw_net.PrepareNetwork()
        if small_modulus_count == 8:
            got = np.asarray(net.GetNext().Decrypt()).reshape(-1)
            want = np.asarray(raw_net.GetNext().Decrypt()).reshape(-1)
            assert np.allclose(got, want, rtol=1e-9, atol=1e-9) and got.argmax() == want.argmax()
        else:
            ma, mb = _compare_layerwise(net, raw_net, rd, rrd, upto=-1)  # everything but the last dense layer
            assert np.allclose(np.asarray(ma.Decrypt()), np.asarray(mb.Decrypt()), rtol=1e-9, atol=1e-9)
            budget = min(f.engine.noise_budget(v.vec, ch, 0) for v in ma.vectors for ch in range(2))
            assert 0 < budget < _last_layer_needs(f, 16384)
    finally:
        f.Dispose()


@pytest.mark.parametrize("small_modulus_count", [9, 8])
def test_lola_cifar_scores_equal_raw_backend(small_modulus_count):
    """LoLa-CIFAR (LolaCifarCryptoNet.cs:27-131; BASELINE config 4) on one synthetic 3x32x32 image with synthetic weights of the
    shipped shapes: 192-column im2col input, 83-map convolution, square, the 5488 x 16268 row-major dense layer (batched
    multiply_plain + rotate-and-sum + one-hot masks, ForceDenseFormat), square, dense 5488 -> 10.  As for LoLa-Dense, the reference's
    SmallModulusCount=8 leaves ~25 bits before the last 16384-slot MultiplyPlain (~55 bits): compared through the second square
    there, and end to end with one more prime."""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import CIFAR_PRIMES, lola_cifar, synthetic_cifar
    from cryptonets_b200.raw import RawFactory
    f = B200BfvFactory(CIFAR_PRIMES, 16384, DecompositionBitCount=60, GaloisDecompositionBitCount=60,
                       SmallModulusCount=small_modulus_count, seed=5)
    try:
        imgs = synthetic_cifar(1)
        net, rd = lola_cifar(f, imgs)
        net.PrepareNetwork()
        raw_net, rrd = lola_cifar(RawFactory(16384), imgs)
        raw_net.PrepareNetwork()
        if small_modulus_count == 9:
            got = np.asarray(net.GetNext().Decrypt()).reshape(-1)
            want = np.asarray(raw_net.GetNext().Decrypt()).reshape(-1)
            assert np.allclose(got, want, rtol=1e-9, atol=1e-9) and got.argmax() == want.argmax()
        else:
            ma, mb = _compare_layerwise(net, raw_net, rd, rrd, upto=-1)
            assert np.allclose(np.asarray(ma.Decrypt()), np.asarray(mb.Decrypt()), rtol=1e-9, atol=1e-9)
            budget = min(f.engine.noise_budget(v.vec, ch, 0) for v in ma.vectors for ch in range(2))
            assert 0 < budget < _last_layer_needs(f, 16384)
    finally:
        f.Dispose()


@pytest.mark.parametrize("small_modulus_count", [8, 7])
def test_lola_large_scores_equal_raw_backend(small_modulus_count):
    """Large LoLa (LoLaCryptonets.cs:330-409; 3 plaintext primes, N=16384, w=60) with synthetic weights of the shipped shapes: 83-map
    8x8 convolution on un-normalised pixels, square, 2608 x 11952 row-major dense layer (ForceDenseFormat), square, dense -> 10.
    Same budget situation as LoLa-Dense / CIFAR: end to end with one more prime than the reference's SmallModulusCount=7, layer by layer
    through the second square with 7."""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import LOLA_LARGE_PRIMES, lola_large, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    f = B200BfvFactory(LOLA_LARGE_PRIMES, 16384, DecompositionBitCount=60, GaloisDecompositionBitCount=60,
                       SmallModulusCount=small_modulus_count, seed=5)
    try:
        imgs = synthetic_mnist(1, seed=3)
        net, rd = lola_large(f, imgs)
        net.PrepareNetwork()
        raw_net, rrd = lola_large(RawFactory(16384), imgs)
        raw_net.PrepareNetwork()
        if small_modulus_count == 8:
            got = np.asarray(net.GetNext().Decrypt()).reshape(-1)
            want = np.asarray(raw_net.GetNext().Decrypt()).reshape(-1)
            assert np.allclose(got, want, rtol=1e-9, atol=1e-9) and got.argmax() == want.argmax()
        else:
            ma, mb = _compare_layerwise(net, raw_net, rd, rrd, upto=-1)
            assert np.allclose(np.asarray(ma.Decrypt()), np.asarray(mb.Decrypt()), rtol=1e-9, atol=1e-9)
            budget = min(f.engine.noise_budget(v.vec, ch, 0) for v in ma.vectors for ch in range(3))
            assert 0 < budget < _last_layer_needs(f, 16384)
    finally:
        f.Dispose()


def test_operation_counts_match_the_reference_call_sequence():
    """The library counts evaluator-level operations the way the reference's OperationsCount does (AtomicSealBfvVector.cs:211-294).  For
    LoLa-small the counts per inference follow from the reference's code alone:
      LLPoolLayer   (5 maps x 25 taps, LLPoolLayer.cs:112-137 -> DenseMatrixBySparseVectorMultiply :466-505): one monomial MultiplyPlain per
                    non-zero tap, one AddMany and one AddPlain per map;
      LLVectorize   (Stack of 5 x 169 slots, Interleave :600-722): vectors 1..4 are rotated by 169 k (NAF hops of 169, 338, 507, 676 =
                    4 + 4 + 3 + 4 = 15 key switches), one AddMany of 5 items;
      Square        one Multiply + one Relinearize;
      LLDenseLayer  (10 rows, EncryptedSealBfvMatrix.cs:79-89 -> DotProduct :964-977): per row one dense MultiplyPlain, SumAllSlots over 8192
                    slots = RotateColumns + 12 RotateRows and 13 Adds (:888-931), one AddPlain for the bias vector;
    all per plaintext modulus (P = 2)."""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import LOLA_SMALL_PRIMES, lola_small, lola_small_weights, synthetic_mnist
    f = B200BfvFactory(LOLA_SMALL_PRIMES, 8192, DecompositionBitCount=40, GaloisDecompositionBitCount=40, SmallModulusCount=4, seed=5)
    try:
        net, rd = lola_small(f, synthetic_mnist(1, seed=6))
        net.PrepareNetwork()
        chain = _layer_chain(net)
        m = rd.GetNext()
        m = chain[1].Apply(m)  # EncryptLayer
        f.engine.op_counts(reset=True)
        per_layer = {}
        for layer in chain[2:]:
            m = layer.Apply(m)
            per_layer[type(layer).__name__] = f.engine.op_counts(reset=True)
        P = 2
        w0 = np.rint(np.asarray(lola_small_weights()["Weights_0"]) * 64)
        taps = sum(int((w0[k * 26:k * 26 + 25] % t != 0).sum()) for k in range(5) for t in LOLA_SMALL_PRIMES)
        c = per_layer["LLPoolLayer"]
        assert (c["ScalarMultiplication"], c["AddMany"], c["AddManyItemCount"], c["PlainAddition"]) == (taps, 5 * P, taps, 5 * P)
        c = per_layer["LLVectorizeLayer"]
        naf_hops = lambda s: sum(1 for _ in _naf(s))
        assert c["Rotation"] == P * sum(naf_hops(169 * k) for k in range(1, 5)) and c["AddMany"] == P and c["AddManyItemCount"] == 5 * P
        assert c["PlainMultiplication"] == 0  # 845 slots < N/2: no vector straddles the half boundary, no mask multiply
        c = per_layer["SquareActivation"]
        assert (c["Multiplication"], c["Relinarization"]) == (P, P)
        c = per_layer["LLDenseLayer"]
        assert (c["PlainMultiplication"], c["ColumnRotation"], c["Rotation"], c["Addition"], c["PlainAddition"]) == (10 * P, 10 * P, 120 * P, 130 * P, 10 * P)
    finally:
        f.Dispose()


def _naf(value):
    """non-adjacent form of a rotation amount (SEAL util::naf): the hops rotate_rows takes when no key for the exact step exists"""
    v, i = abs(value), 0
    while v:
        z = (2 - (v & 3)) if (v & 1) else 0
        v = (v - z) >> 1
        if z:
            yield z * (1 << i)
        i += 1
