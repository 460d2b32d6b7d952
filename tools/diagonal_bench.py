"""LoLa-Large and LoLa-CIFAR with their big ForceDenseFormat dense layer (dense4) on the row method, the diagonal method and the diagonal
method with diagonals held in NTT form (diagonal_ntt, --ntt-bytes of them; default the whole matrix), alternated.

Per network and method: device time per image (every layer synchronised), the dense4 layer's time (after one untimed dense4
call), key switches per image from the
operation counters (row-rotation hops + column rotations + relinearisations), and for the diagonal methods the prepare time, the
coefficient-form and NTT-form bytes the prepared matrix holds, dense4 at B = 8 inputs in one call and the device time of one more dense4
call per profiler family at B = 1 and at B = 8 (cnhe_prof_collect; the lift is booked as "other", the MAC as "scalar_mac_layer", whose
algorithmic bytes over its time give dense4_mac_GBps and dense4_B8_mac_GBps).  held_bytes is the prepared matrix's device_bytes (both
forms), coeff_bytes / ntt_bytes its parts.  Full residency takes about 39 GB for LoLa-CIFAR and 46 GB for LoLa-Large: run one network
per process.  Then the diagonal method at the reference's SmallModulusCount: whether the scores decrypt, and the budget entering the last layer.  --score-methods alternates the Method of the score layer (dense6: "rows", the
reference's, and / or "folded") within every dense4 method; each record has dense6's time, its key switches and the bytes of the score
ciphertexts.  Prints one JSON line per measurement (and writes them to --out if given)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cryptonets_b200 import networks as nw  # noqa: E402
from cryptonets_b200._lib import CnheError  # noqa: E402
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


def mem_used_mb():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=memory.used", "--format=csv,noheader,nounits"], capture_output=True, text=True)
        return int(q.stdout.split()[0])
    except (OSError, ValueError, IndexError):
        return None


def profile(eng, call):
    """Device time per profiler family of one call that returns a list of outputs (cnhe_prof_collect), and the diagonal MAC's
    ("scalar_mac_layer") algorithmic HBM bytes over its device time."""
    eng.sync()
    eng.prof_enable(True)
    outs = call()
    eng.sync()
    fam = eng.prof_collect()
    eng.prof_enable(False)
    for o in outs:
        o.Dispose()
    mac = fam["scalar_mac_layer"]
    return {k: round(v["ms"], 3) for k, v in fam.items()}, (round(mac["bytes"] / mac["ms"] / 1e6, 1) if mac["ms"] else None)


def run(f, name, method, imgs, batch8, ntt_bytes=None, score_method="rows"):
    """method: rows, diagonal or diagonal_ntt."""
    eng = f.engine
    diag = method != "rows"
    eng.set_option("release_cached_memory", 1)  # the previous arm's scratch goes back to the driver before this arm's matrix
    kw = dict(diag_ntt_bytes=ntt_bytes) if method == "diagonal_ntt" else {}
    net, rd = getattr(nw, name)(f, imgs, dense_method="diagonal" if diag else "rows", score_method=score_method, **kw)
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
    held = coeff_held = ntt_held = None
    if diag:
        ntt_held = layers[D].DiagonalMatrix.NttInfo()["bytes"]
        held = layers[D].DiagonalMatrix.Info()["device_bytes"]
        coeff_held = held - ntt_held
    mem_after_prepare = mem_used_mb()
    m = rd.GetNext()
    eng.op_counts(reset=True)
    total, dense4, dense6, ks6 = 0.0, 0.0, 0.0, 0
    for i, L in enumerate(layers[1:], 1):
        if i == D:  # one untimed dense4 first: its scratch comes from the driver once, not inside the timed call
            L.Apply(m).Dispose()
        if i == len(layers) - 1:
            ks6 = key_switches(eng.op_counts())
        eng.sync()
        t0 = time.perf_counter()
        m2 = L.Apply(m)
        eng.sync()
        dt = time.perf_counter() - t0
        total += dt
        if i == len(layers) - 1:
            dense6 = dt
            ks6 = key_switches(eng.op_counts()) - ks6
        if i == D:
            dense4 = dt
            x4 = m  # dense4's input (kept for the batched call)
        elif m is not m2 and i != D + 1:
            m.Dispose()
        m = m2
    ks = key_switches(eng.op_counts())
    score_bytes = sum(v.vec.blocks for v in m.vectors) * eng.P * 2 * len(eng.q) * eng.N * 8
    rec = dict(net=name, method=method, score_method=score_method, k=len(eng.q), s_per_image=total, dense4_s=dense4, dense6_s=dense6,
               dense6_key_switches=ks6, score_bytes=score_bytes, key_switches=ks, prepare_s=prep,
               held_bytes=held, coeff_bytes=coeff_held, ntt_bytes=ntt_held, device_mem_used_mb_after_prepare=mem_after_prepare)
    if diag:
        rec["dense4_families_ms"], rec["dense4_mac_GBps"] = profile(eng, lambda: [layers[D].Apply(x4)])
    if batch8 and diag:
        eng.sync()
        t0 = time.perf_counter()
        outs = layers[D].ApplyBatch([x4] * 8)
        eng.sync()
        rec["dense4_B8_s"] = time.perf_counter() - t0
        for o in outs:
            o.Dispose()
        rec["dense4_B8_families_ms"], rec["dense4_B8_mac_GBps"] = profile(eng, lambda: layers[D].ApplyBatch([x4] * 8))
    scores = np.asarray(m.Decrypt()).reshape(-1)
    net.DisposeNetwork()
    return rec, scores


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nets", default="lola_large,lola_cifar")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--skip-reference-count", action="store_true", help="skip the runs at the reference's SmallModulusCount")
    ap.add_argument("--ntt-bytes", type=int, default=None, help="diagonal_ntt's budget in bytes (default: the whole matrix; LoLa-Large "
                    "wholly resident ran out of memory on an 80 GB H100; 34359738368 = 32 GiB works)")
    ap.add_argument("--methods", default="rows,diagonal,diagonal_ntt")
    ap.add_argument("--score-methods", default="rows")
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
            for method in a.methods.split(","):
                for score_method in a.score_methods.split(","):
                    try:
                        rec, got = run(f, name, method, imgs, batch8=True, ntt_bytes=a.ntt_bytes, score_method=score_method)
                    except CnheError as e:  # e.g. a budget the card cannot hold next to the rest of the network
                        rec = dict(net=name, method=method, score_method=score_method, rep=rep, error=str(e), device_mem_used_mb=mem_used_mb())
                        recs.append(rec)
                        print(json.dumps(rec), flush=True)
                        continue
                    rec["rep"] = rep
                    rec["scores_equal_raw"] = bool(np.allclose(got, want, rtol=1e-9, atol=1e-9))
                    recs.append(rec)
                    print(json.dumps(rec), flush=True)
        f.Dispose()
        if a.skip_reference_count:
            continue
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
