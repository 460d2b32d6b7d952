"""Host-side planner of the wgmma scalar-MAC kernel (csrc/vec.cu: umma_try / umma_search), through the library's planner probe -- no GPU
needed.  A bundle is at most 128 outputs whose taps lie in a window of consecutive inputs; the planner tries every bundle size and keeps
the plan with the fewest 32-tap chunks per tile that fits in shared memory; identical weight matrices are stored once."""
import ctypes as C

import numpy as np
import pytest


@pytest.fixture(scope="module")
def probe():
    from cryptonets_b200 import _lib
    fn = _lib.lib().cnhe_debug_mac_plan
    fn.restype = C.c_int
    fn.argtypes = [C.POINTER(C.c_int32), C.POINTER(C.c_double), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]

    def run(gather, w, limbs=6):
        g = np.ascontiguousarray(gather, dtype=np.int32)
        ww = np.ascontiguousarray(w, dtype=np.float64)
        out = (C.c_int * 4)()
        ok = fn(g.ctypes.data_as(C.POINTER(C.c_int32)), ww.ctypes.data_as(C.POINTER(C.c_double)), g.shape[0], g.shape[1], limbs, out)
        return None if not ok else dict(bundles=out[0], chunks=out[1], weight_bytes=out[2], extra_taps=out[3])
    return run


def conv_gather(side, ker, stride, pad, maps):
    osz = (side + pad - ker) // stride + 1
    rows = []
    for y in range(osz):
        for x in range(osz):
            row = [-1] * (ker * ker)
            for dy in range(ker):
                for dx in range(ker):
                    iy, ix = y * stride + dy - pad, x * stride + dx - pad
                    if 0 <= iy < side and 0 <= ix < side:
                        row[dy * ker + dx] = iy * side + ix
            rows += [row] * maps
    return np.array(rows, dtype=np.int32), osz


def test_cryptonets_convolution_plan(probe):
    """CryptoNets' first layer (28x28, 5x5 kernel, stride 2, upper padding 1, 5 maps; CryptoNets.cs:40-48): one bundle per output row (65
    outputs), 5 chunks each except the padded top row (4 input rows -> 4 chunks); the 12 interior rows share ONE weight matrix."""
    gather, osz = conv_gather(28, 5, 2, 1, 5)
    assert osz == 13 and gather.shape == (845, 25)
    rng = np.random.default_rng(1)
    kern = rng.integers(-67, 68, (5, 25)).astype(np.float64)
    w = np.tile(kern, (osz * osz, 1))
    w[gather < 0] = 0
    plan = probe(gather, w)
    assert plan == dict(bundles=13, chunks=64, weight_bytes=9 * 4096, extra_taps=0)


def test_dense_plan_with_wide_weights(probe):
    """845 -> 100: one bundle of 27 chunks; the weights beyond a signed byte ride on one extra chunk of W2 columns (one per tap that has such
    a weight in any row).  A weight beyond +-254 has no plan (the caller falls back)."""
    M, K = 100, 845
    rng = np.random.default_rng(2)
    w = rng.integers(-127, 128, (M, K)).astype(np.float64)
    cols = rng.choice(K, 31, replace=False)
    for c in cols:
        w[rng.integers(0, M), c] = rng.choice([-165, 140, 254, -254])
    gather = np.tile(np.arange(K, dtype=np.int32), (M, 1))
    assert probe(gather, w) == dict(bundles=1, chunks=28, weight_bytes=28 * 4096, extra_taps=31)
    w[3, 7] = 300
    assert probe(gather, w) is None
    # a layer whose window does not fit next to the rings in shared memory (K = 1600: 50 chunks of weights = 200 KB) has no plan either
    K2 = 1600
    assert probe(np.tile(np.arange(K2, dtype=np.int32), (16, 1)), rng.integers(-5, 6, (16, K2)).astype(np.float64)) is None


def test_small_layers_and_ragged_groups(probe):
    """more outputs per gather row than one MMA holds -> no plan; a stride-1 convolution packs several output rows per bundle"""
    gather = np.tile(np.arange(40, dtype=np.int32), (130, 1))
    assert probe(gather, np.ones((130, 40))) is None
    gather, osz = conv_gather(9, 3, 1, 0, 2)
    w = np.ones(gather.shape)
    plan = probe(gather, w)
    assert plan is not None and plan["bundles"] == 1 and plan["chunks"] == 3 and plan["extra_taps"] == 0  # 98 outputs, window = all 81 inputs
