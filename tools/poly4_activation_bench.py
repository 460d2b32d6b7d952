"""Cubic / quartic activation benchmark: device-event time per call of cnhe_layer_poly at degrees 3 and 4, of two chained
cnhe_layer_square calls (the least the quartic can cost: two multiplicative levels of squares), and of the compositions a caller builds
today from public calls, alternated in one process, plus the per-family device times of one profiled call of each.

The compositions: x^2 = layer_square(x), x^3 = x^2 . x (a product of two distinct ciphertexts: the separate product kernels), x^4 =
layer_square(x^2), then one scalar multiply per term and one add per term -- each a pass over the ciphertexts, one call per vector.  Their
words differ from cnhe_layer_poly's (different circuits); the cost is what is compared.

Shapes as in poly_activation_bench.py: "cryptonets" = the CryptoNets square (945 ciphertexts in one vector, N = 8192, k = 5, one
plaintext prime); "lola_small_b32" = lola_small's square for B = 32 clients (32 one-ciphertext vectors, N = 8192, k = 3, two plaintext
primes).  One JSON line per shape and round, with the card's name, power limit and maximum SM clock."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from cryptonets_b200.engine import DENSE, SPARSE, Engine
from poly_activation_bench import SHAPES, card


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
        cs = [eng.plain(np.array([v]), 1.0, SPARSE) for v in (7.0, -5.0, 3.0, 2.0, 1.0)]  # x^0 .. x^4
        const = eng.plain(np.full(dim, 7.0), 1.0, DENSE)  # add_plain of the constant to every block

        def poly(d):
            return lambda: eng.layer_poly(xs, cs[:d + 1])

        def two_squares():
            x2 = eng.layer_square(xs)
            out = eng.layer_square(x2)
            for v in x2:
                v.dispose()
            return out

        def composition(d):
            def run():
                x2 = eng.layer_square(xs)
                x4 = eng.layer_square(x2) if d == 4 else None
                out = []
                for i, x in enumerate(xs):
                    powers = [x, x2[i], eng.pointwise_multiply(x2[i], x)] + ([x4[i]] if d == 4 else [])
                    acc, tmp = None, []
                    for j, p in enumerate(powers, 1):
                        term = eng.pointwise_multiply(p, cs[j])
                        tmp.append(term)
                        acc = term if acc is None else eng.add(acc, term)
                        tmp.append(acc)
                    out.append(eng.add(acc, const))
                    tmp.append(powers[2])
                    for v in {id(v): v for v in tmp}.values():
                        v.dispose()
                for v in x2 + (x4 or []):
                    v.dispose()
                return out
            return run

        variants = {"poly_d4": poly(4), "poly_d3": poly(3), "two_squares": two_squares, "composition_d4": composition(4),
                    "composition_d3": composition(3)}
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
