"""Where dense4's device time goes on the diagonal method: the profiler families (cnhe_prof_collect) and, in a run of its own, the
kernels by name (torch.profiler, CUDA activities).  One JSON line per network.

    python tools/dense4_split.py [nets, default lola_cifar,lola_large] [DiagonalNttBytes, default 0]"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import diagonal_bench as db  # noqa: E402
from cryptonets_b200 import networks as nw  # noqa: E402
from cryptonets_b200.he import B200BfvFactory  # noqa: E402


def main():
    nets = sys.argv[1] if len(sys.argv) > 1 else "lola_cifar,lola_large"
    ntt_bytes = int(sys.argv[2]) if len(sys.argv) > 2 else 0
    print(json.dumps(dict(gpu=db.gpu_info())), flush=True)
    for name in nets.split(","):
        primes, kref, mk = db.NETS[name]
        imgs = mk()
        f = B200BfvFactory(primes, 16384, DecompositionBitCount=60, GaloisDecompositionBitCount=60, SmallModulusCount=kref + 1, seed=5)
        eng = f.engine
        net, rd = getattr(nw, name)(f, imgs, dense_method="diagonal", diag_ntt_bytes=ntt_bytes)
        net.PrepareNetwork()
        layers = db.chain(net)
        m = rd.GetNext()
        for L in layers[1:5]:
            m = L.Apply(m)
        D = layers[5]
        times = []
        for _ in range(4):
            eng.sync()
            t0 = time.perf_counter()
            y = D.Apply(m)
            eng.sync()
            times.append(time.perf_counter() - t0)
            y.Dispose()
        eng.prof_enable(True)
        y = D.Apply(m)
        eng.sync()
        fam = eng.prof_collect()
        eng.prof_enable(False)
        y.Dispose()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as p:
            y = D.Apply(m)
            eng.sync()
        y.Dispose()
        kern = {}
        for ev in p.key_averages():
            us = getattr(ev, "device_time_total", None)
            if us is None:
                us = ev.cuda_time_total
            if us > 0:
                kern[ev.key[:90]] = dict(ms=us / 1e3, n=ev.count)
        kern = dict(sorted(kern.items(), key=lambda kv: -kv[1]["ms"]))
        print(json.dumps(dict(net=name, k=len(eng.q), ntt_bytes=ntt_bytes, dense4_s=times, families=fam, kernels=kern)), flush=True)
        net.DisposeNetwork()
        f.Dispose()


if __name__ == "__main__":
    main()
