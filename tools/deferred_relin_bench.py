"""Deferred relinearisation benchmark: one CryptoNets-MNIST batch (8192 images, N = 8192, the reference's two plaintext primes) through
the default network and through cryptonets_mnist(defer_relinearization=True), alternated in one process.

Per arm and round: device-event time of one batch (network.GetNext: encryption, every layer, the scores); once per arm: the per-family
device times of one profiled batch (cnhe_prof_collect), the relinearisations per plaintext prime per batch (cnhe_op_counts), the scores'
noise budget and whether the decrypted scores equal the default arm's.  One JSON line per round, then a summary line, each with the card's
name, power limit and maximum SM clock."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from cryptonets_b200.he import B200BfvFactory
from cryptonets_b200.networks import CRYPTONETS_PRIMES, cryptonets_mnist, synthetic_mnist
from poly_activation_bench import card


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8192)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    c = card()
    f = B200BfvFactory(CRYPTONETS_PRIMES, 8192, seed=77)
    eng = f.engine
    imgs = synthetic_mnist(args.images, seed=3)
    arms = {}
    for name, defer in (("default", False), ("deferred", True)):
        net, _ = cryptonets_mnist(f, imgs, timing=False, defer_relinearization=defer)
        net.PrepareNetwork()
        net.GetNext().Dispose()  # warm-up: module loads, MAC plans, pools
        arms[name] = net
    summary = {"card": c, "images": args.images, "P": len(CRYPTONETS_PRIMES), "k": eng.k, "arms": {}}
    scores = {}
    for name, net in arms.items():
        eng.sync()
        eng.op_counts(reset=True)
        out = net.GetNext()
        relin = eng.op_counts(reset=True)["Relinarization"] // len(CRYPTONETS_PRIMES)
        budget = min(eng.noise_budget(v.vec, ch, 0) for v in out.vectors for ch in range(eng.P))
        scores[name] = np.asarray(out.Decrypt())
        out.Dispose()
        eng.sync()
        eng.prof_enable(True)
        net.GetNext().Dispose()
        eng.sync()
        prof = eng.prof_collect()
        eng.prof_enable(False)
        summary["arms"][name] = {"relinearizations_per_prime": relin, "score_noise_budget_bits": budget,
                                 "families_ms": {k_: round(p["ms"], 3) for k_, p in prof.items() if p["ms"] > 0}, "ms_per_batch": []}
    summary["scores_equal"] = bool(np.array_equal(scores["default"], scores["deferred"]))
    for r in range(args.rounds):
        res = {"round": r, "card": c, "ms_per_batch": {}}
        for name, net in arms.items():
            eng.sync()
            eng.timer_start()
            out = net.GetNext()
            res["ms_per_batch"][name] = round(eng.timer_stop_ms(), 3)
            out.Dispose()
            summary["arms"][name]["ms_per_batch"].append(res["ms_per_batch"][name])
        print(json.dumps(res), flush=True)
    print(json.dumps(summary), flush=True)
    f.Dispose()


if __name__ == "__main__":
    main()
