"""Output-noise bounds of the networks for sanitisation (DESIGN 4.18; networks.OUTPUT_NOISE_BITS): each network at the parameters of its
end-to-end GPU test (tools/level_bench.py NETS, CryptoNets-MNIST at N = 8192), one eager inference per seed, and for a sample of its output
ciphertexts the exact noise polynomial, computed with the secret key and big integers (tests/sanitize_ref.py noise_poly on the CPU
oracle's transforms).  Prints, per network, the largest infinity norm in bits over the seeds, the smallest final noise budget, and whether
a flood of e + margin + 40 + log2 N bits fits (at most floor(log2(q/t)) - 2 bits: the budget must exceed about 40 + log2 N + margin + 2);
when it does not, how many bits and coefficient primes (at the network's average prime width) are missing.

usage: python tools/output_noise.py [--seeds 5 6 7] [--nets lola_small lola ...] [--out output_noise.json]"""
import argparse
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import level_bench as B  # noqa: E402
import sanitize_ref as sr  # noqa: E402
from cryptonets_b200 import networks as nw  # noqa: E402
from cryptonets_b200.he import B200BfvFactory  # noqa: E402
from oracle.oracle_py import Oracle  # noqa: E402

LAMBDA = 40


def build(name, seed):
    """(factory, output matrix, dbc) of one eager inference"""
    if name == "cryptonets_mnist":
        f = B200BfvFactory(nw.CRYPTONETS_PRIMES, 8192, seed=seed)
        net, _ = nw.cryptonets_mnist(f, nw.synthetic_mnist(16, seed=6), batch_size=16, timing=False)
        net.PrepareNetwork()
        return f, net.GetNext(), (10, 20)
    base, k = (name[:-3], 5) if name == "lola_small_k5" else (name, None)
    f = B.factory(base, seed=seed)
    if k:  # lola_small on one coefficient prime more than its test parameters (k = 4): the parameters whose budget covers lambda = 40
        _, primes, N, (w, wg), _, _ = B.NETS[base]
        f.Dispose()
        f = B200BfvFactory(primes, N, DecompositionBitCount=w, GaloisDecompositionBitCount=wg, SmallModulusCount=k, seed=seed)
    imgs = B.NETS[base][5]()
    net, _ = B.NETS[base][0](f, imgs)
    net.PrepareNetwork()
    x = B.encrypted_input(f, base, imgs)
    m = x
    for layer in B.chain_of(net):
        o = layer.Apply(m)
        if m is not x and o is not m:
            m.Dispose()
        m = o
    return f, m, B.NETS[base][3]


def measure(name, seed, sample):
    f, m, dbc = build(name, seed)
    eng = f.engine
    vecs = [v.vec for v in m.vectors]
    idx = sorted(set(np.linspace(0, len(vecs) - 1, min(sample, len(vecs))).astype(int)))
    raw = eng.export_raw_many([vecs[i] for i in idx])
    worst, budget = 0, 10 ** 9
    for c, t in enumerate(eng.primes):
        orc = Oracle(t, eng.N, eng.k, dbc[0], dbc[1], custom_q=eng.q)
        orc.keygen(seed + c)
        for j, i in enumerate(idx):
            noise, _ = sr.noise_poly(orc, raw[c, j, 0])
            worst = max(worst, max(abs(e) for e in noise))
            budget = min(budget, eng.noise_budget(vecs[i], c, 0))
    out = dict(N=eng.N, k=eng.k, noise_bits=math.log2(worst) if worst else 0.0, budget=budget, max_flood_bits=eng.sanitize_max_bits(),
               avg_prime_bits=sum(x.bit_length() for x in eng.q) / eng.k)
    m.Dispose()
    f.Dispose()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, nargs="+", default=[5, 6, 7])
    ap.add_argument("--nets", nargs="+", default=["lola_small", "lola", "lola_dense", "lola_large", "lola_cifar", "cryptonets_mnist"])
    ap.add_argument("--sample", type=int, default=4)
    ap.add_argument("--margin", type=int, default=nw.OUTPUT_NOISE_MARGIN)
    ap.add_argument("--out", default=None, help="also write the full results as JSON to this file")
    a = ap.parse_args()
    res = {}
    for name in a.nets:
        runs = [measure(name, s, a.sample) for s in a.seeds]
        e = max(r["noise_bits"] for r in runs)
        bound = int(math.ceil(e)) + a.margin
        budget = min(r["budget"] for r in runs)
        N = runs[0]["N"]
        flood = bound + LAMBDA + int(math.log2(N))
        deficit = max(0, flood - runs[0]["max_flood_bits"])  # the flood must fit below q / 4t (cnhe_vecs_sanitize's limit)
        res[name] = dict(runs=runs, noise_bits=e, bound=bound, budget=budget, flood_bits=flood, covers=deficit == 0, deficit_bits=deficit,
                         extra_primes=int(math.ceil(deficit / runs[0]["avg_prime_bits"])))
        print(json.dumps({name: {k: v for k, v in res[name].items() if k != "runs"}}), flush=True)
    if not a.out:
        return
    with open(a.out, "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
