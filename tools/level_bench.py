"""Levels on an H100 (DESIGN 4.17): trace the noise budgets of each LoLa network at its full level, plan a schedule, and time the networks
with and without it.

  python tools/level_bench.py trace [--nets a,b]   per named layer, the smallest budget over sampled ciphertexts and every plaintext
                                                   channel; tools/level_plan.py's schedule from them; the final budget
  python tools/level_bench.py bench [--nets a,b] [--rounds 3]
      for each network with a committed schedule (networks.LEVEL_SCHEDULES), alternated with the unswitched network over the rounds:
      time per image and per layer (host clock around work that ends in a synchronise of every context of the family), the key-switch
      family's device-event time (a separate profiled pass), the device bytes of the keys at each level, and the switch kernel's time and
      HBM rate against 3.35 TB/s; with the card's name, power limit and maximum SM clock.
Results go to stdout, and with --out to a JSON file.  Parameters: those of each network's end-to-end GPU test
(tests/test_gpu_network.py): one prime more than the reference's SmallModulusCount on the row method, LoLa at its default modulus."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import level_plan  # noqa: E402
from cryptonets_b200 import networks as nw  # noqa: E402
from cryptonets_b200.he import B200BfvFactory  # noqa: E402
from cryptonets_b200.interfaces import EMatrixFormat  # noqa: E402
from cryptonets_b200.layers import EncryptLayer, TimingLayer  # noqa: E402

HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s

# network: (builder, plaintext primes, N, decomposition bit counts, coefficient primes, images)
NETS = {
    "lola_small": (nw.lola_small, nw.LOLA_SMALL_PRIMES, 8192, (40, 40), 4, lambda: nw.synthetic_mnist(1, seed=6)),
    "lola": (nw.lola, nw.LOLA_PRIMES, 8192, (10, 20), 5, lambda: nw.synthetic_mnist(1, seed=6)),
    "lola_dense": (nw.lola_dense, nw.LOLA_DENSE_PRIMES, 16384, (60, 60), 8, lambda: nw.synthetic_mnist(1, seed=6)),
    "lola_large": (nw.lola_large, nw.LOLA_LARGE_PRIMES, 16384, (60, 60), 8, lambda: nw.synthetic_mnist(1, seed=6)),
    "lola_cifar": (nw.lola_cifar, nw.CIFAR_PRIMES, 16384, (60, 60), 9, lambda: nw.synthetic_cifar(1, seed=6)),
}


def factory(name, seed=5):
    _, primes, N, (w, wg), k, _ = NETS[name]
    return B200BfvFactory(primes, N, DecompositionBitCount=w, GaloisDecompositionBitCount=wg, SmallModulusCount=k, seed=seed)


def family(f):
    """the factory and every level factory made from it"""
    out = [f]
    for g in f.__dict__.get("_levels", {}).values():
        out += family(g)
    return out


def sync(f):
    for g in family(f):
        g.engine.sync()


def chain_of(net):
    layers, layer = [], net
    while not isinstance(layer, EncryptLayer):
        if not isinstance(layer, TimingLayer):
            layers.append(layer)
        layer = layer.Source
    layers.reverse()
    for layer in layers:
        if not layer.layerPrepared:
            layer.Prepare()
            layer.layerPrepared = True
    return layers


def encrypted_input(f, net_name, imgs):
    _, reader = NETS[net_name][0](f, imgs)
    m = reader.GetNext()
    x = f.GetEncryptedMatrix(m.Data, EMatrixFormat.ColumnMajor, 1)
    x.RegisterScale(m.Scale)
    return x


def min_budgets(m, sample=32):
    """per plaintext channel, the smallest budget over up to `sample` vectors of m (evenly spaced) and their first and last blocks"""
    vs = m.vectors if hasattr(m, "vectors") else [m]
    idx = sorted(set(np.linspace(0, len(vs) - 1, min(sample, len(vs))).astype(int)))
    eng = vs[0].factory.engine
    out = []
    for ch in range(eng.P):
        b = 1 << 30
        for i in idx:
            v = vs[i].vec
            for blk in sorted({0, v.blocks - 1}):
                b = min(b, eng.noise_budget(v, ch, blk))
        out.append(b)
    return out


def run(layers, x, per_layer=None, f=None):
    """the layers on x (kept); per_layer: a list that gets each layer's seconds (a synchronise of the family after every layer)"""
    m = x
    for layer in layers:
        t0 = time.perf_counter()
        o = layer.Apply(m)
        if per_layer is not None:
            sync(f)
            per_layer.append(time.perf_counter() - t0)
        if m is not x and o is not m:
            m.Dispose()
        m = o
    return m


def trace(name):
    f = factory(name)
    try:
        imgs = NETS[name][5]()
        net, _ = NETS[name][0](f, imgs)
        layers = chain_of(net)
        x = encrypted_input(f, name, imgs)
        m, rows = x, []
        for layer in layers:
            o = layer.Apply(m)
            if m is not x and o is not m:
                m.Dispose()
            m = o
            if getattr(layer, "LevelName", None):
                rows.append([layer.LevelName, min_budgets(m)])
        final = min_budgets(m)
        e = f.engine
        rec = dict(N=e.N, q=e.q, primes=e.primes, dbc=NETS[name][3][0], dbc_galois=NETS[name][3][1], mtilde_centered=0, layers=rows)
        return dict(net=name, k=e.k, layers=rows, final=final, plan=level_plan.plan(rec), schedule=level_plan.schedule(rec))
    finally:
        f.Dispose()


def key_bytes(e):
    kN = e.k * e.N
    return 8 * e.P * (kN + 2 * kN + e.relin_digits * 2 * kN + e.n_galois * e.galois_digits * 2 * kN)


def switch_rate(f, k2, n=64, reps=20):
    e, lvl = f.engine, f.AtLevel(k2).engine
    vs = e.encrypt_many(np.zeros((n, e.N)))
    for o in e.mod_switch(vs, lvl):
        o.dispose()
    sync(f)
    t0 = time.perf_counter()
    for _ in range(reps):
        lvl.dispose_many(e.mod_switch(vs, lvl))
    sync(f)
    s = (time.perf_counter() - t0) / reps
    nbytes = n * 2 * (e.k + k2) * e.N * 8 * e.P
    e.dispose_many(vs)
    return dict(ciphertexts=n * e.P, k=e.k, k_out=k2, ms=s * 1e3, bytes=nbytes, GBps=nbytes / s / 1e9, frac_of_peak=nbytes / s / HBM_PEAK)


def bench(name, rounds):
    levels = nw.LEVEL_SCHEDULES.get(name)
    if not levels:
        return dict(net=name, schedule=None, note="no committed schedule: nothing to compare")
    f = factory(name)
    try:
        imgs = NETS[name][5]()
        chains = {"full": chain_of(NETS[name][0](f, imgs)[0]), "levels": chain_of(NETS[name][0](f, imgs, levels=levels)[0])}
        x = encrypted_input(f, name, imgs)
        for c in chains.values():  # warm-up: every shape, plan and level
            run(c, x).Dispose()
        sync(f)
        times = {k: [] for k in chains}
        layer_times = {k: [] for k in chains}
        for _ in range(rounds):
            for key, c in chains.items():
                t0 = time.perf_counter()
                out = run(c, x)
                sync(f)
                times[key].append(time.perf_counter() - t0)
                out.Dispose()
                per = []
                run(c, x, per, f).Dispose()
                layer_times[key].append(per)
        ks = {}
        for key, c in chains.items():
            for g in family(f):
                g.engine.prof_enable(True)
            run(c, x).Dispose()
            sync(f)
            ks[key] = sum(g.engine.prof_collect()["keyswitch_mac"]["ms"] for g in family(f))
            for g in family(f):
                g.engine.prof_enable(False)
        names = {key: [type(l).__name__ + ("(%s)" % l.LevelName if getattr(l, "LevelName", None) else "") for l in c] for key, c in chains.items()}
        return dict(net=name, schedule=levels,
                    ms_per_image={k: float(np.median(v)) * 1e3 for k, v in times.items()},
                    ms_rounds={k: [t * 1e3 for t in v] for k, v in times.items()},
                    ms_per_layer={k: list(zip(names[k], (np.median(np.array(v), axis=0) * 1e3).tolist())) for k, v in layer_times.items()},
                    keyswitch_ms=ks,
                    key_bytes={g.engine.k: key_bytes(g.engine) for g in family(f)},
                    switch=switch_rate(f, min(levels.values())))
    finally:
        f.Dispose()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", choices=["trace", "bench"])
    ap.add_argument("--nets", default=",".join(NETS))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card(), results=[])
    for name in a.nets.split(","):
        r = trace(name) if a.mode == "trace" else bench(name, a.rounds)
        res["results"].append(r)
        print(json.dumps(r), flush=True)
    print("card:", res["card"])
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
