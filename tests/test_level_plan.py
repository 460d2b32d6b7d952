"""The level planner (tools/level_plan.py) and the `levels` argument of the networks on the Raw backend.  CPU only."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import level_plan as L  # noqa: E402

Q16 = [0xfffffffd8001, 0xfffffffa0001, 0xfffffff00001, 0x1fffffff68001, 0x1fffffff50001, 0x1ffffffee8001, 0x1ffffffea0001, 0x1ffffffe88001]


def _rec(layers, primes=(34359771137, 34360754177), q=Q16):
    return dict(N=16384, q=list(q), primes=list(primes), dbc=60, dbc_galois=60, mtilde_centered=0, layers=layers)


def test_lola_dense_trace_ladder():
    """LoLa-Dense at k = 8 (profiles/r02_noise_trace.md): the budgets 221, 169, 125, 85 after the first square, the packed dense layer,
    the second square and the interleave give 8 -> 7 -> 6 -> 5 -> 4 with the 7-bit margin, the floors about 244, 195, 146 and 98"""
    rec = _rec([["act4", [221, 221]], ["dense6", [169, 169]], ["act7", [125, 125]], ["inter8", [85, 85]]])
    m = L.models(rec)[0]
    assert [round(L.level_floor(m, k, 60, 60)) for k in (7, 6, 5, 4)] == [244, 195, 146, 98]
    assert L.plan(rec) == [("act4", 7), ("dense6", 6), ("act7", 5), ("inter8", 4)]
    assert L.schedule(rec) == {"act4": 7, "dense6": 6, "act7": 5, "inter8": 4}


def test_levels_never_rise_and_a_binding_floor_keeps_the_level():
    # a budget that grows again (a layer after a fresh-looking one) must not raise the level; 240 + 7 > 243.8 keeps all 8 primes
    rec = _rec([["a", [240, 240]], ["b", [100, 100]], ["c", [230, 230]], ["d", [150, 150]]])
    assert L.plan(rec) == [("a", 8), ("b", 5), ("c", 5), ("d", 5)]  # floors at 5 and 4 primes: 146.2 and 97.5
    assert L.schedule(_rec([["a", [240, 240]]])) == {}
    # exactly at the floor minus the margin: the level drops; a tenth of a bit more and it does not
    f7 = min(L.level_floor(m, 7, 60, 60) for m in L.models(_rec([])))
    assert L.plan(_rec([["a", [f7 - L.MARGIN, f7 - L.MARGIN]]]))[0][1] == 7
    assert L.plan(_rec([["a", [f7 - L.MARGIN + 0.1, f7 - L.MARGIN + 0.1]]]))[0][1] == 8


def test_the_noisiest_channel_decides():
    one = L.plan(_rec([["a", [120, 120]]]))[0][1]
    assert L.plan(_rec([["a", [120, 200]]]))[0][1] > one
    assert L.plan(_rec([["a", [200, 120]]]))[0][1] == L.plan(_rec([["a", [200, 200]]]))[0][1]
    # a larger plaintext prime raises every floor's noise: the same budget needs at least as many primes
    assert L.plan(_rec([["a", [120, 120]]], primes=(34359771137, 1 << 50)))[0][1] >= one


def test_switch_rounding_term():
    from noise_model import Model
    m = L.models(_rec([]))[0]
    # c sqrt(N / 18) t / q': 2.19 + 4.92 + log2 t - log2 q' bits
    assert abs(m.switch_peak(300.0) - (np.log2(m.c) + 0.5 * np.log2(16384 / 18.0) + np.log2(34359771137) - 300.0)) < 1e-9
    assert Model.budget(m.switch_peak(300.0)) == pytest.approx(300.0 - np.log2(34359771137) - np.log2(m.c * np.sqrt(16384 / 18.0)) - 1)


@pytest.mark.parametrize("net", ["lola", "lola_dense", "lola_small"])
def test_levels_on_the_raw_backend_change_nothing(net):
    from cryptonets_b200 import networks as nw
    from cryptonets_b200.raw import RawFactory
    levels = {"lola": {"act3": 4, "act7": 3}, "lola_dense": {"act4": 7, "dense6": 6, "act7": 5, "inter8": 4}, "lola_small": {"act3": 2}}[net]
    imgs = nw.synthetic_mnist(1, seed=2)
    outs = []
    for lv in (None, levels):
        n, _ = getattr(nw, net)(RawFactory(16384 if net == "lola_dense" else 8192), imgs, levels=lv)
        n.PrepareNetwork()
        outs.append(np.asarray(n.GetNext().Decrypt()))
    assert np.array_equal(outs[0], outs[1])


def test_levels_name_only_known_layers():
    from cryptonets_b200 import networks as nw
    from cryptonets_b200.raw import RawFactory
    with pytest.raises(ValueError, match="act9"):
        nw.lola(RawFactory(8192), nw.synthetic_mnist(1), levels={"act9": 3})
