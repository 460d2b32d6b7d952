"""Client-side cost of values entering and leaving ciphertexts (DESIGN 4.19): encryption of the CryptoNets-MNIST input batch (784 x 8192
values, N = 8192, P = 2) and of one lola_small im2col matrix, and decryption of the 10 x 8192 scores, per call, each ending in a device
synchronise.  Paths: encrypt / encrypt_compact from numpy and from a CUDA tensor, decrypt to numpy and to a CUDA tensor.

  python tools/client_bench.py [--rounds 3] [--reps 5] [--parent DIR] [--out results/client_bench.json]

--parent DIR: a package directory (DIR/cryptonets_b200) of another build whose host-array calls are timed in alternation with this
build's, in separate processes, `--rounds` times.  The card, its power limit and clocks are recorded with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CN_PRIMES = [549764251649, 549764284417]
LOLA_PRIMES = [2277377, 2424833]


def card():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def measure(reps):
    """one process: every path of the build on sys.path, median ms per call"""
    import numpy as np
    import torch
    from cryptonets_b200.engine import Engine
    dev_paths = hasattr(Engine, "_device_rows")
    res = {}

    def timed(name, fn):
        fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
            if isinstance(out, list):
                out[0].eng.dispose_many(out)
        res[name] = sorted(ts)[len(ts) // 2]

    rng = np.random.default_rng(0)
    for label, primes, count, shape in (("cryptonets", CN_PRIMES, -1, (784, 8192)), ("lola_small", LOLA_PRIMES, 3, (1, 8192))):
        eng = Engine(primes, 8192, 10, 20, count)
        eng.keygen(1)
        x = rng.integers(0, 256, shape).astype(np.float64)
        xt = torch.from_numpy(x).cuda()
        timed(label + "/encrypt_numpy", lambda: eng.encrypt_many(x, 1.0))
        timed(label + "/encrypt_compact_numpy", lambda: eng.encrypt_compact(x, 1.0))
        if dev_paths:
            timed(label + "/encrypt_tensor", lambda: eng.encrypt_many(xt, 1.0))
            timed(label + "/encrypt_compact_tensor", lambda: eng.encrypt_compact(xt, 1.0))
        if label == "cryptonets":
            scores = eng.encrypt_many(rng.integers(-10 ** 6, 10 ** 6, (10, 8192)).astype(np.float64), 1.0)
            timed("cryptonets/decrypt_numpy", lambda: eng.decrypt_many(scores))
            if dev_paths:
                timed("cryptonets/decrypt_tensor", lambda: eng.decrypt_many(scores, device=True))
            eng.dispose_many(scores)
        eng.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--parent", default=None)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        print(json.dumps(measure(a.reps)))
        return
    builds = [("this", ROOT)] + ([("parent", os.path.abspath(a.parent))] if a.parent else [])
    rows = {b: [] for b, _ in builds}
    for _ in range(a.rounds):
        for b, path in builds:
            env = dict(os.environ, PYTHONPATH=path)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--reps", str(a.reps)], env=env, cwd=path,
                               capture_output=True, text=True)
            if p.returncode:
                sys.exit("%s build failed (%d):\n%s" % (b, p.returncode, p.stderr[-3000:]))
            rows[b].append(json.loads(p.stdout.strip().splitlines()[-1]))
    result = {"card": card(), "rounds": a.rounds, "reps": a.reps, "ms": {}}
    for b, runs in rows.items():
        result["ms"][b] = {k: sorted(r[k] for r in runs) for k in runs[0]}
    text = json.dumps(result, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(text)


if __name__ == "__main__":
    main()
