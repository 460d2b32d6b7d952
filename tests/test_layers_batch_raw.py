"""On the Raw backend every LoLa layer's ApplyBatch equals one Apply per matrix (the batched device paths fall back there)."""
import numpy as np

from cryptonets_b200.layers import EncryptLayer
from cryptonets_b200.networks import lola, lola_dense, synthetic_mnist
from cryptonets_b200.raw import RawFactory


def _chain(net):
    chain, layer = [], net
    while not isinstance(layer, EncryptLayer):
        chain.append(layer)
        layer = layer.Source
    return chain[::-1], layer


def test_ll_layers_apply_batch_equals_apply_per_matrix():
    imgs = synthetic_mnist(3, seed=14)
    seen = set()
    for build, n in ((lola, 8192), (lola_dense, 16384)):
        net, reader = build(RawFactory(n), imgs)
        net.PrepareNetwork()
        chain, enc = _chain(net)
        ms = [enc.Apply(reader.GetNext()) for _ in range(len(imgs))]
        for layer in chain:
            batched = layer.ApplyBatch(ms)
            single = [layer.Apply(m) for m in ms]
            assert len(batched) == len(single)
            for a, b in zip(batched, single):
                assert np.array_equal(np.asarray(a.Decrypt()), np.asarray(b.Decrypt())), type(layer).__name__
            seen.add(type(layer).__name__)
            ms = single
    assert {"LLDuplicateLayer", "LLPackedDenseLayer", "LLInterleaveLayer", "LLInterleavedDenseLayer", "LLPreConvLayer"} <= seen
