"""Level planner: the coefficient primes each layer of a network needs (ModSwitchLayer, DESIGN 4.17), from the noise budgets an
inference at the full level leaves after each layer.  CPU only; the noise formulas are tools/noise_model.py's Model.

Rule.  At each layer boundary, in network order, take the smallest k' (never above the previous boundary's) for which, on every plaintext
channel, the level's three floors -- the budget a relinearisation and a Galois key switch leave on a noiseless ciphertext at q' = q_0 ..
q_{k'-1}, and the budget the switch's own rounding leaves -- are all at least the budget there plus `margin`.  A ciphertext whose budget is
`margin` bits below a floor loses at most log2(1 + 2^-margin) bits to that noise source; a chain of m key switches, each adding its
floor's noise to a ciphertext at least that much noisier, loses at most log2(1 + m 2^-margin).  The default margin, 7 bits, keeps a chain
of 64 key switches within 0.6 bit, so a schedule leaves the final budget within about a bit of the unswitched run's.

usage: python tools/level_plan.py budgets.json
  budgets.json: {"N", "q", "primes", "dbc", "dbc_galois", "mtilde_centered", "layers": [[name, [budget per channel]], ...]}"""
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from noise_model import Model  # noqa: E402

MARGIN = 7.0


def models(rec):
    return [Model(rec, ch) for ch in range(len(rec["primes"]))]


def level_floor(m, k, dbc, dbc_galois):
    """the smallest of the three floors (budgets) of one channel's model at the prefix of k primes"""
    q = m.q[:k]
    logq = math.log2(math.prod(q))
    return min(Model.budget(m.ks_peak(dbc, q)), Model.budget(m.ks_peak(dbc_galois, q)), Model.budget(m.switch_peak(logq)))


def plan(rec, margin=MARGIN):
    """[(layer, k')] for every boundary of rec["layers"]: k' primes from that layer's output on"""
    ms = models(rec)
    k = len(rec["q"])
    out = []
    for name, budgets in rec["layers"]:
        while k > 1 and all(level_floor(m, k - 1, rec["dbc"], rec["dbc_galois"]) >= b + margin for m, b in zip(ms, budgets)):
            k -= 1
        out.append((name, k))
    return out


def schedule(rec, margin=MARGIN):
    """the `levels` argument of the network: the boundaries where the level drops"""
    full, levels, prev = len(rec["q"]), {}, len(rec["q"])
    for name, k in plan(rec, margin):
        if k < prev:
            levels[name] = k
        prev = k
    return levels if prev < full else {}


if __name__ == "__main__":
    rec = json.load(open(sys.argv[1]))
    for name, k in plan(rec):
        print("%-10s k' = %d" % (name, k))
    print("levels =", schedule(rec) or "none: no boundary clears a smaller level")
