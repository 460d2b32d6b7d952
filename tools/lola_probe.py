"""Exploratory: LoLa / LoLa-Dense on the GPU backend vs the Raw backend, with per-layer timings and remaining noise budget."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from cryptonets_b200.he import B200BfvFactory
from cryptonets_b200.networks import (CIFAR_PRIMES, LOLA_DENSE_PRIMES, LOLA_PRIMES, lola, lola_cifar, lola_dense, synthetic_cifar,
                                      synthetic_mnist)
from cryptonets_b200.raw import RawFactory


def chain(net):
    out, p = [], net
    while p is not None and hasattr(p, "Apply") and getattr(p, "Source", None) is not None:
        out.append(p)
        p = p.Source
    return out[::-1]


which = sys.argv[1] if len(sys.argv) > 1 else "lola"
imgs = synthetic_mnist(1, seed=6)
if which == "lola":
    f = B200BfvFactory(LOLA_PRIMES, 8192, seed=5)
    build, block = lola, 8192
elif which == "cifar":
    imgs = synthetic_cifar(1)
    f = B200BfvFactory(CIFAR_PRIMES, 16384, DecompositionBitCount=60, GaloisDecompositionBitCount=60, SmallModulusCount=8, seed=5)
    build, block = lola_cifar, 16384
else:
    f = B200BfvFactory(LOLA_DENSE_PRIMES, 16384, DecompositionBitCount=60, GaloisDecompositionBitCount=60, SmallModulusCount=7, seed=5)
    build, block = lola_dense, 16384
net, rd = build(f, imgs)
t0 = time.time(); net.PrepareNetwork(); print("prepare %.2fs" % (time.time() - t0))
rnet, rrd = build(RawFactory(block), imgs)
rnet.PrepareNetwork()
ma, mb = rd.GetNext(), rrd.GetNext()
for A, B in zip(chain(net), chain(rnet)):
    t0 = time.time()
    ma2 = A.Apply(ma); f.engine.sync()
    dt = time.time() - t0
    mb2 = B.Apply(mb)
    da, db = np.asarray(ma2.Decrypt()), np.asarray(mb2.Decrypt())
    ok = da.shape == db.shape and np.allclose(da, db, rtol=1e-9, atol=1e-9)
    try:
        budget = min(f.engine.noise_budget(v.vec, ch, 0) for v in ma2.vectors for ch in range(f.engine.P))
    except Exception as e:
        budget = str(e)[:40]
    print("%-24s %.3fs cols=%d equal=%s budget=%s" % (type(A).__name__, dt, ma2.ColumnCount, ok, budget), flush=True)
    ma, mb = ma2, mb2
print("scores", np.asarray(ma.Decrypt()).ravel()[:10])
print("raw   ", np.asarray(mb.Decrypt()).ravel()[:10])
f.Dispose()
