"""Cost of sanitisation (cnhe_vecs_sanitize, DESIGN 4.18) on the GPU: device time per call for n = 1, 10, 128 and 945 ciphertexts next to
cnhe_vecs_encrypt of the same count, the finish kernel's algorithmic bytes over its time (profiling family 6), and the replayed inference
of lola_small and LoLa with and without a final SanitizeLayer, alternated over three rounds.  Prints the card name, power limit and
maximum SM clock of the run.  Needs a CUDA device.

usage: python tools/sanitize_bench.py [--reps 20] [--out sanitize_bench.json]"""
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

from cryptonets_b200 import networks as nw  # noqa: E402
from cryptonets_b200.engine import Engine  # noqa: E402
from cryptonets_b200.layers import EncryptLayer, SanitizeLayer  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip()


def timed(eng, fn, reps):
    fn()  # warm-up
    eng.sync()
    t0 = time.perf_counter()
    for _ in range(reps):
        r = fn()
    eng.sync()
    return (time.perf_counter() - t0) / reps * 1e3, r


def calls(reps):
    """lola_small's parameters (N = 8192, k = 4, two plaintext primes): per-call time of sanitize and encrypt, and the finish kernel"""
    eng = Engine(nw.LOLA_SMALL_PRIMES, 8192, 40, 40, 4)
    eng.keygen(1)
    b = 13 + 40 + 10
    rows = []
    for n in (1, 10, 128, 945):
        vals = np.random.default_rng(n).integers(-50, 50, (n, 100)).astype(np.float64)
        vecs = eng.encrypt_many(vals)
        ms_s, out = timed(eng, lambda: eng.sanitize(vecs, b), reps)
        eng.dispose_many(out)
        ms_e, out = timed(eng, lambda: eng.encrypt_many(vals), reps)
        eng.dispose_many(out)
        eng.prof_enable(True)
        out = eng.sanitize(vecs, b)
        eng.sync()
        pf = eng.prof_collect()["sanitize_finish"]
        ms_k, nbytes = pf["ms"], pf["bytes"]
        eng.prof_enable(False)
        eng.dispose_many(out + vecs)
        rows.append(dict(n=n, sanitize_ms=ms_s, encrypt_ms=ms_e, finish_kernel_ms=ms_k, finish_bytes=nbytes,
                         finish_GBps=nbytes / (ms_k * 1e-3) / 1e9 if ms_k else None))
        print(json.dumps(rows[-1]), flush=True)
    eng.close()
    return rows


def _chain(net):
    chain, layer = [], net
    while not isinstance(layer, EncryptLayer):
        chain.append(layer)
        layer = layer.Source
    return layer, chain


def inference(name, reps):
    """replayed inference time with and without a final SanitizeLayer (flood of log2 N + 40 bits), alternated over three rounds"""
    import level_bench as B
    res = {"plain": [], "sanitized": []}
    caps = {}
    for kind in res:
        f = B.factory(name)
        imgs = B.NETS[name][5]()
        net, reader = B.NETS[name][0](f, imgs)
        if kind == "sanitized":
            net = SanitizeLayer(Source=net, NoiseBits=0, StatisticalBits=40)
        net.PrepareNetwork()
        x = _chain(net)[0].Apply(reader.GetNext())
        caps[kind] = (f, f.CaptureInference(net, x), x)
    for _ in range(3):
        for kind, (f, cap, x) in caps.items():
            ms, _ = timed(f.engine, lambda: cap.Run(x), reps)
            res[kind].append(ms)
    for f, cap, _ in caps.values():
        cap.Dispose()
        f.Dispose()
    print(json.dumps({name: res}), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the full results as JSON to this file")
    a = ap.parse_args()
    res = dict(card=card())
    print(res["card"], flush=True)
    res["calls"] = calls(a.reps)
    res["inference"] = {n: inference(n, a.reps) for n in ("lola_small", "lola")}
    if not a.out:
        return
    with open(a.out, "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
