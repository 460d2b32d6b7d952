"""Randomised cross-check of the wgmma scalar-MAC kernel against the FP64 scalar-MAC kernel (both on the GPU, bit-exact expected):
random dense shapes and random strided/padded convolutions over a slab of ciphertexts, weights up to +-254, random biases.
usage: python tools/umma_stress.py [cases] [seed]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from cryptonets_b200.engine import Engine, DENSE, SPARSE



def run(cases, seed, log=print):
  """returns the number of cases whose outputs differ between the two kernels"""
  rng = np.random.default_rng(seed)
  eng = Engine([40961], 4096, 10, 20, -1)
  eng.keygen(7)
  N = eng.N
  q = np.array(eng.q, dtype=np.uint64)
  bad = 0
  for case in range(cases):
      if case % 2 == 0:  # dense
          M, K = int(rng.integers(8, 129)), int(rng.integers(32, 260))
          n_in = K + int(rng.integers(0, 3))
          gather = np.tile(np.arange(K, dtype=np.int32), (M, 1))
          if rng.random() < 0.5:  # a rotated window of the slab, still one gather row for all outputs
              gather = (gather + int(rng.integers(0, n_in - K + 1))).astype(np.int32)
          w = rng.integers(-127, 128, (M, K)).astype(np.float64)
          desc = "dense %dx%d" % (M, K)
      else:  # convolution
          side, ker, stride, pad, maps = int(rng.integers(6, 15)), int(rng.integers(2, 5)), int(rng.integers(1, 3)), int(rng.integers(0, 2)), int(rng.integers(1, 7))
          osz = (side + pad - ker) // stride + 1
          n_in, K, M = side * side, ker * ker, maps * osz * osz
          gather = np.full((M, K), -1, dtype=np.int32)
          w = np.zeros((M, K))
          kern = rng.integers(-127, 128, (maps, K)).astype(np.float64)
          m = 0
          for y in range(osz):
              for x in range(osz):
                  for f in range(maps):
                      for dy in range(ker):
                          for dx in range(ker):
                              iy, ix = y * stride + dy - pad, x * stride + dx - pad
                              if 0 <= iy < side and 0 <= ix < side:
                                  gather[m, dy * ker + dx] = iy * side + ix
                      w[m] = kern[f]
                      m += 1
          w[gather < 0] = 0
          keep = (w != 0).any(axis=1)
          if not keep.all():
              continue
          desc = "conv %dx%d k%d s%d p%d maps%d -> %d outputs" % (side, side, ker, stride, pad, maps, M)
      if rng.random() < 0.5:  # some weights beyond one signed byte
          for _ in range(int(rng.integers(1, 6))):
              i, j = int(rng.integers(0, M)), int(rng.integers(0, K))
              if gather[i, j] >= 0:
                  w[i, j] = int(rng.choice([-254, -200, -128, 128, 165, 254]))
      cts = rng.integers(0, 1 << 62, (n_in, 2, eng.k, N), dtype=np.uint64) % q[None, None, :, None]
      cts[0] = (q - 1)[None, :, None]
      ins = eng.import_raw_many(cts.reshape(n_in, -1), n_in, 1, N, 4.0)
      bias = rng.integers(-1000, 1000, M).astype(np.float64)
      wv = [eng.plain(w[i], 1.0, SPARSE) for i in range(M)]
      bv = [eng.plain(np.full(N, bias[i]), 4.0, DENSE) for i in range(M)]
      os.environ.pop("CNHE_MAC_NO_UMMA", None)
      a = eng.layer_conv_dense(ins, gather, wv, bv, M, K)
      os.environ["CNHE_MAC_NO_IMMA"] = "1"
      b = eng.layer_conv_dense(ins, gather, wv, bv, M, K)
      del os.environ["CNHE_MAC_NO_IMMA"]
      diff = sum(not np.array_equal(a[i].export_raw(0, 0), b[i].export_raw(0, 0)) for i in range(M))
      bad += diff > 0
      log("%-50s %s" % (desc, "ok" if diff == 0 else "MISMATCH in %d outputs" % diff))
  eng.close()
  return bad


if __name__ == "__main__":
    n_bad = run(int(sys.argv[1]) if len(sys.argv) > 1 else 24, int(sys.argv[2]) if len(sys.argv) > 2 else 5)
    print("cases with a mismatch:", n_bad)
    sys.exit(1 if n_bad else 0)
