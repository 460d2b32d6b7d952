"""LoLa-Large and LoLa-CIFAR with their big ForceDenseFormat dense layer (dense4) on the row method and on the diagonal method, alternated.

Per network and method: device time per image (every layer synchronised), the dense4 layer's time, key switches per image from the
operation counters (row-rotation hops + column rotations + relinearisations), and for the diagonal method the prepare time, the bytes the
prepared matrix holds and dense4 at B = 8 inputs in one call.  Then the diagonal method at the reference's SmallModulusCount: whether the
scores decrypt, and the budget entering the last layer.  Prints one JSON line per measurement (and writes them to --out if given)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cryptonets_b200 import networks as nw  # noqa: E402
from cryptonets_b200.he import B200BfvFactory  # noqa: E402
from cryptonets_b200.raw import RawFactory  # noqa: E402

NETS = {"lola_large": (nw.LOLA_LARGE_PRIMES, 7, lambda: nw.synthetic_mnist(1, seed=3)),
        "lola_cifar": (nw.CIFAR_PRIMES, 8, lambda: nw.synthetic_cifar(1))}


def gpu_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def chain(net):
    out, p = [], net
    while p is not None and hasattr(p, "Source"):
        out.append(p)
        p = p.Source
    return out[::-1]


def key_switches(c):
    return c["Rotation"] + c["ColumnRotation"] + c["Relinarization"]


def run(f, name, method, imgs, batch8):
    eng = f.engine
    net, rd = getattr(nw, name)(f, imgs, dense_method=method)
    layers = chain(net)
    D = 5  # reader, encrypt, pool, vectorize, square, dense4, square, dense
    for L in layers[1:]:
        if L is not layers[D]:
            L.Prepare()
            L.layerPrepared = True
    eng.sync()
    t0 = time.perf_counter()
    layers[D].Prepare()
    layers[D].layerPrepared = True
    eng.sync()
    prep = time.perf_counter() - t0
    held = layers[D].DiagonalMatrix.Info()["device_bytes"] if method == "diagonal" else None
    m = rd.GetNext()
    eng.op_counts(reset=True)
    total, dense4 = 0.0, 0.0
    for i, L in enumerate(layers[1:], 1):
        eng.sync()
        t0 = time.perf_counter()
        m2 = L.Apply(m)
        eng.sync()
        dt = time.perf_counter() - t0
        total += dt
        if i == D:
            dense4 = dt
            x4 = m  # dense4's input (kept for the batched call)
        elif m is not m2 and i != D + 1:
            m.Dispose()
        m = m2
    ks = key_switches(eng.op_counts())
    rec = dict(net=name, method=method, k=len(eng.q), s_per_image=total, dense4_s=dense4, key_switches=ks, prepare_s=prep, held_bytes=held)
    if batch8 and method == "diagonal":
        eng.sync()
        t0 = time.perf_counter()
        outs = layers[D].ApplyBatch([x4] * 8)
        eng.sync()
        rec["dense4_B8_s"] = time.perf_counter() - t0
        for o in outs:
            o.Dispose()
    scores = np.asarray(m.Decrypt()).reshape(-1)
    net.DisposeNetwork()
    return rec, scores


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nets", default="lola_large,lola_cifar")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    recs = [dict(gpu=gpu_info())]
    print(json.dumps(recs[0]), flush=True)
    for name in a.nets.split(","):
        primes, kref, mk = NETS[name]
        imgs = mk()
        raw, _ = getattr(nw, name)(RawFactory(16384), imgs)
        raw.PrepareNetwork()
        want = np.asarray(raw.GetNext().Decrypt()).reshape(-1)
        f = B200BfvFactory(primes, 16384, DecompositionBitCount=60, GaloisDecompositionBitCount=60, SmallModulusCount=kref + 1, seed=5)
        for rep in range(a.reps):
            for method in ("rows", "diagonal"):
                rec, got = run(f, name, method, imgs, batch8=rep == 0)
                rec["rep"] = rep
                rec["scores_equal_raw"] = bool(np.allclose(got, want, rtol=1e-9, atol=1e-9))
                recs.append(rec)
                print(json.dumps(rec), flush=True)
        f.Dispose()
        # the reference's SmallModulusCount on the diagonal method: budget entering the last layer and whether the scores decrypt
        f = B200BfvFactory(primes, 16384, DecompositionBitCount=60, GaloisDecompositionBitCount=60, SmallModulusCount=kref, seed=5)
        for method in ("rows", "diagonal"):
            net, rd = getattr(nw, name)(f, imgs, dense_method=method)
            net.PrepareNetwork()
            m = rd.GetNext()
            for L in chain(net)[1:-1]:
                m = L.Apply(m)
            budget = min(f.engine.noise_budget(v.vec, ch, 0) for v in m.vectors for ch in range(f.engine.P))
            got = np.asarray(chain(net)[-1].Apply(m).Decrypt()).reshape(-1)
            rec = dict(net=name, method=method, k=kref, budget_into_last_layer=budget,
                       scores_equal_raw=bool(np.allclose(got, want, rtol=1e-9, atol=1e-9)))
            recs.append(rec)
            print(json.dumps(rec), flush=True)
            net.DisposeNetwork()
        f.Dispose()
    if a.out:
        with open(a.out, "w") as fh:
            for r in recs:
                fh.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
