"""Encrypted x encrypted column-major product: cnhe_mat_mul_colmajor_sparse (a multiply and relinearisation per product, then a sum) against
cnhe_mat_mul_colmajor_sparse_deferred (products summed in the NTT domain, one floor per chunk, one relinearisation per output block),
alternated in one process.

Shapes: K encrypted columns of one block (N = 8192, the CryptoNets coefficient primes, the reference's two plaintext primes) times an
encrypted sparse vector of dimension K, for each --K.  Per shape and round: device-event time of one call of each arm.  Once per arm and
shape: per-family device times, launches and booked bytes of one profiled call (cnhe_prof_collect), the relinearisations per plaintext
prime (cnhe_op_counts), the polynomial transforms per plaintext prime those counts imply (per product 4 (k + kb) forward and 3 (k + kb)
inverse for the existing call; per distinct input 2 (k + kb) forward and per output block and chunk 3 (k + kb) inverse for the deferred
one; per key switch D k forward and 2 k inverse), whether both arms decrypt to the same values and their noise budgets.  One JSON line per round, then a summary line per shape, each with the card's name, power limit and maximum SM clock."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from cryptonets_b200.engine import DENSE, SPARSE, Engine
from cryptonets_b200.networks import CRYPTONETS_PRIMES
from poly_activation_bench import card


def transforms(eng, arm, K, counts):
    kt, P = eng.k + eng.kb, eng.P
    mul, ks = counts["Multiplication"] // P, counts["Relinarization"] // P
    if arm == "existing":
        fwd, inv = mul * 2 * 2 * kt, mul * 3 * kt
    else:
        chunks = -(-K // eng.product_sum_terms())
        fwd, inv = (mul + K) * 2 * kt, ks * chunks * 3 * kt
    return {"forward": fwd + ks * eng.relin_digits * eng.k, "inverse": inv + ks * 2 * eng.k}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--K", type=int, nargs="+", default=[100, 845])
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    c = card()
    eng = Engine(CRYPTONETS_PRIMES, 8192, 10, 20, -1)
    eng.keygen(5)
    P, N = eng.P, eng.N
    arms = {"existing": eng.mat_mul_colmajor_sparse, "deferred": eng.mat_mul_colmajor_sparse_deferred}
    for K in args.K:
        rng = np.random.default_rng(K)
        cols = [eng.encrypt(rng.integers(-60, 60, N).astype(np.float64), 1.0, DENSE) for _ in range(K)]
        sparse = eng.encrypt(rng.integers(-60, 60, K).astype(np.float64), 1.0, SPARSE)
        summary = {"card": c, "N": N, "k": eng.k, "kb": eng.kb, "P": P, "K": K, "blocks": 1, "K_c": eng.product_sum_terms(), "arms": {}}
        vals = {}
        for name, fn in arms.items():
            fn(cols, sparse).dispose()  # warm-up: module loads, pools
            eng.sync()
            eng.op_counts(reset=True)
            out = fn(cols, sparse)
            counts = eng.op_counts(reset=True)
            vals[name] = eng.decrypt(out)
            budget = min(eng.noise_budget(out, ch, 0) for ch in range(P))
            out.dispose()
            eng.sync()
            eng.prof_enable(True)
            fn(cols, sparse).dispose()
            eng.sync()
            prof = eng.prof_collect()
            eng.prof_enable(False)
            summary["arms"][name] = {
                "relinearizations_per_prime": counts["Relinarization"] // P, "multiplications_per_prime": counts["Multiplication"] // P,
                "transforms_per_prime": transforms(eng, name, K, counts),
                "noise_budget_bits": budget,
                "families": {f: {"ms": round(p["ms"], 3), "launches": p["launches"]} for f, p in prof.items() if p["launches"]},
                "ms_per_call": []}
        summary["values_equal"] = bool(np.array_equal(vals["existing"], vals["deferred"]))
        for r in range(args.rounds):
            res = {"round": r, "K": K, "card": c, "ms_per_call": {}}
            for name, fn in arms.items():
                eng.sync()
                eng.timer_start()
                out = fn(cols, sparse)
                res["ms_per_call"][name] = round(eng.timer_stop_ms(), 3)
                out.dispose()
                summary["arms"][name]["ms_per_call"].append(res["ms_per_call"][name])
            print(json.dumps(res), flush=True)
        print(json.dumps(summary), flush=True)
        for v in cols + [sparse]:
            v.dispose()
    eng.close()


if __name__ == "__main__":
    main()
