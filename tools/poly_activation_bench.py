"""Quadratic-activation benchmark: device-event time per call of cnhe_layer_poly2, cnhe_layer_square and the composition a caller builds
today from public calls, alternated in one process, plus the per-family device times of one profiled call of each.

The composition: layer_square (multiply + relinearise), then multiply by the plain scalar A, multiply x by B, add, add_plain C -- four
more passes over the ciphertexts (one call each per vector).  Its words differ from poly2's (A is applied after the key switch, so the
key switch's noise is scaled by A); the cost is what is compared.

Shapes: "cryptonets" = the CryptoNets square (945 ciphertexts in one vector, N = 8192, k = 5, one plaintext prime); "lola_small_b32" =
lola_small's square for B = 32 clients (32 one-ciphertext vectors, N = 8192, k = 3, two plaintext primes).  One JSON line per shape and
round, with the card's name, power limit and maximum SM clock."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from cryptonets_b200.engine import DENSE, SPARSE, Engine

SHAPES = {
    "cryptonets": dict(t=[549764251649], count=-1, dbc=10, n_vecs=1, blocks=945),
    "lola_small_b32": dict(t=[2277377, 2424833], count=3, dbc=40, n_vecs=32, blocks=1),
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().split("\n")[0]
        return [s.strip() for s in q.split(",")]
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    c = card()
    for name in args.shapes.split(","):
        cfg = SHAPES[name]
        eng = Engine(cfg["t"], 8192, cfg["dbc"], cfg["dbc"], cfg["count"])
        eng.keygen(1)
        rng = np.random.default_rng(0)
        dim = 8192 * cfg["blocks"]
        xs = [eng.encrypt(rng.integers(-50, 50, dim).astype(np.float64), 1.0, DENSE) for _ in range(cfg["n_vecs"])]
        a, b, cc = (eng.plain(np.array([v]), 1.0, SPARSE) for v in (3.0, -5.0, 7.0))
        cw = eng.plain(np.full(dim, 7.0), 1.0, DENSE)  # add_plain of C to every block (a sparse scalar adds to one-block vectors only)

        def poly2():
            return eng.layer_poly2(xs, a, b, cc)

        def square():
            return eng.layer_square(xs)

        def composition():
            out = []
            for x, s in zip(xs, eng.layer_square(xs)):
                t1, t2 = eng.pointwise_multiply(s, a), eng.pointwise_multiply(x, b)
                t3 = eng.add(t1, t2)
                out.append(eng.add(t3, cw))
                for v in (s, t1, t2, t3):
                    v.dispose()
            return out

        variants = dict(poly2=poly2, square=square, composition=composition)
        for fn in variants.values():  # warm-up: every shape and path of the timed window
            for v in fn():
                v.dispose()
        eng.sync()
        for r in range(args.rounds):
            res = {"shape": name, "round": r, "ciphertexts_per_channel": cfg["n_vecs"] * cfg["blocks"], "channels": len(cfg["t"]), "k": eng.k,
                   "ms_per_call": {}, "families_ms": {}, "card": c}
            for vname, fn in variants.items():
                eng.sync()
                eng.timer_start()
                for _ in range(args.iters):
                    for v in fn():
                        v.dispose()
                res["ms_per_call"][vname] = round(eng.timer_stop_ms() / args.iters, 3)
            if r == 0:
                for vname, fn in variants.items():
                    eng.sync()
                    eng.prof_enable(True)
                    for v in fn():
                        v.dispose()
                    eng.sync()
                    prof = eng.prof_collect()
                    eng.prof_enable(False)
                    res["families_ms"][vname] = {k_: round(p["ms"], 3) for k_, p in prof.items() if p["ms"] > 0}
            print(json.dumps(res), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
