"""he.level_factories: the level factories a recording of a levelled chain enlists (CaptureInference(SpanLevels=True)), on the Raw
backend.  A RawFactory has no levels, so its switches name none; a Raw factory that makes levels (as B200BfvFactory.AtLevel does) names
each level its switches run on once, in chain order."""
from cryptonets_b200.he import level_factories
from cryptonets_b200.networks import LEVEL_SCHEDULES, lola, lola_dense, synthetic_mnist
from cryptonets_b200.raw import RawFactory


class _LevelledRaw(RawFactory):
    """a Raw factory with cached level factories, one per prime count (as B200BfvFactory.AtLevel caches them)"""

    def __init__(self, N, k):
        super().__init__(N)
        self.k = k
        self.made = {}

    def AtLevel(self, k):
        if k == self.k:
            return self
        if k not in self.made:
            self.made[k] = _LevelledRaw(self.BlockSize, k)
        return self.made[k]


def _chain(net):
    from cryptonets_b200.layers import EncryptLayer
    chain, layer = [], net
    while not isinstance(layer, EncryptLayer):
        chain.append(layer)
        layer = layer.Source
    return chain[::-1]


def test_raw_factory_names_no_level():
    net, _ = lola(RawFactory(8192), synthetic_mnist(1, seed=1), levels=LEVEL_SCHEDULES["lola"])
    assert level_factories(_chain(net)) == []


def test_unlevelled_chain_names_no_level():
    net, _ = lola(_LevelledRaw(8192, 5), synthetic_mnist(1, seed=1))
    assert level_factories(_chain(net)) == []


def test_each_level_once_in_chain_order():
    f = _LevelledRaw(8192, 5)
    net, _ = lola(f, synthetic_mnist(1, seed=1), levels=LEVEL_SCHEDULES["lola"])
    got = level_factories(_chain(net))
    assert [g.k for g in got] == [4, 3]
    assert got[0] is f.AtLevel(4) and got[1] is f.AtLevel(4).AtLevel(3)
    f = _LevelledRaw(16384, 8)
    net, _ = lola_dense(f, synthetic_mnist(1, seed=1), levels=LEVEL_SCHEDULES["lola_dense"])
    assert [g.k for g in level_factories(_chain(net))] == [7, 6, 5, 4]


def test_a_switch_to_the_current_level_names_none():
    f = _LevelledRaw(8192, 5)
    net, _ = lola(f, synthetic_mnist(1, seed=1), levels={"dense5": 5, "act7": 4})
    assert [g.k for g in level_factories(_chain(net))] == [4]
