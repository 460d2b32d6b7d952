"""Analytic BFV noise model next to the measured per-operation trace (tools/noise_trace.py), rendered as a markdown report.

Every evaluator-level operation is checked ON ITS OWN: the trace holds, for each operation, the measured invariant noise budget of its
first output AND the budgets its inputs had, so the model predicts the output budget from the measured inputs -- errors do not
accumulate along the network.  The model is the textbook average-case BFV analysis (peak = c * rms with c = sqrt(2 ln 2N)):

  fresh (SEAL 3.2 encrypts Delta*m):   |v| <= (t/2) (q mod t)/q  [rounding term of Delta = floor(q/t)]  +  c (t/q) sigma sqrt(4N/3)
  key switch, digit width w:           v += c (t/q) sigma sqrt(N sum_digits 4^bits/3)          (relinearise, every rotation hop)
  multiply_plain, dense plaintext:     v *= (t/sqrt12) sqrt N                                   (plaintext coefficients uniform mod t)
  multiply_plain, constant w:          v *= |w|;   scalar MAC: v = rss_k(|w_k| v_k)
  ct x ct (BEHZ) + relinearise:        v = t sqrt(N) sqrt((2N/3+1)/12) (v1 + v2)  (+ key switch);   un-centred m~ adds a constant
  add / sub / add_many:                root-sum-square of the inputs

usage: python tools/noise_model.py gpurun_out/noise_trace.json > profiles/r02_noise_trace.md"""
import json
import math
import sys

SIGMA = 3.19


def peak_factor(N):
    return math.sqrt(2.0 * math.log(2.0 * N))


def prod(xs):
    r = 1
    for x in xs:
        r *= int(x)
    return r


class Model:
    def __init__(self, rec, channel):
        self.N = rec["N"]
        self.q = [int(x) for x in rec["q"]]
        self.Q = prod(self.q)
        self.t = int(rec["primes"][channel])
        self.c = peak_factor(self.N)
        self.logq = math.log2(self.Q)
        self.mt = rec["mtilde_centered"]
        self.ks_relin = self.ks_peak(rec["dbc"])
        self.ks_gal = self.ks_peak(rec["dbc_galois"])

    def ks_peak(self, w, q=None):  # log2 of the peak of the key-switching noise (invariant, i.e. times t/q), at q or a prefix of it
        q = self.q if q is None else q
        ss = 0.0
        for p in q:
            bits = p.bit_length()
            sh = 0
            while sh < bits:
                b = min(w, bits - sh)
                ss += 4.0 ** b / 3.0
                sh += w
        rms = SIGMA * math.sqrt(self.N * ss)
        return math.log2(self.c * rms) + math.log2(self.t) - math.log2(prod(q))

    def switch_peak(self, logq_prime):
        """log2 of the peak invariant noise a modulus switch to q' adds: t/q' times the rounding r0 + r1 s, |r_i| <= 1/2 uniform, whose
        coefficients have rms sqrt(1/12 + N (2/3) / 12) ~ sqrt(N / 18)"""
        return math.log2(self.c * math.sqrt(self.N / 18.0)) + math.log2(self.t) - logq_prime

    @staticmethod
    def peak(budget):  # log2 peak from a budget
        return -(budget + 1.0)

    @staticmethod
    def budget(logpeak):
        return -logpeak - 1.0

    @staticmethod
    def rss(*logs):
        m = max(logs)
        return m + 0.5 * math.log2(sum(4.0 ** (x - m) for x in logs))

    def fresh(self):
        r = self.Q % self.t
        p_round = math.log2(self.t / 2.0) + math.log2(r) - self.logq
        p_gauss = math.log2(self.c * SIGMA * math.sqrt(4.0 * self.N / 3.0 + 1.0)) + math.log2(self.t) - self.logq
        return self.budget(math.log2(2.0 ** p_round + 2.0 ** p_gauss)), self.budget(p_round), self.budget(p_gauss)

    def flood_bits(self, noise_bits, statistical_bits=40):
        """The flood width b of a sanitisation (DESIGN 4.18) that hides an output noise of at most 2^noise_bits (infinity norm) within
        statistical distance 2^-statistical_bits over all N coefficients: b = e + lambda + log2 N"""
        return int(noise_bits) + int(statistical_bits) + int(round(math.log2(self.N)))

    def max_flood_bits(self):
        """the widest flood cnhe_vecs_sanitize accepts for this plaintext modulus: floor(log2(q / t)) - 2"""
        return (self.Q // self.t).bit_length() - 1 - 2

    def sanitize(self, b, budget_in):
        """The budget after a sanitisation of flood width b of a ciphertext with budget budget_in, or None when the sum may change the
        plaintext: the input noise, the flood (peak 2^b, uniform) and a fresh encryption's noise add, so the budget is about
        log2(q/t) - b - 1 once the flood dominates.  An input noise of 2^e leaves a budget of about log2(q/t) - e - 1, so the flood of
        flood_bits(e, lambda) fits only while budget_in exceeds about lambda + log2 N + 2 bits."""
        p_flood = b + math.log2(self.t) - self.logq
        p_fresh = math.log2(self.c * SIGMA * math.sqrt(4.0 * self.N / 3.0 + 1.0)) + math.log2(self.t) - self.logq
        out = self.budget(self.rss(self.peak(budget_in), p_flood, p_fresh))
        return out if out > 0 else None

    def plain_gain(self):
        return math.log2(self.t / math.sqrt(12.0)) + 0.5 * math.log2(self.N)

    def mult_gain(self):  # per unit of (v1 + v2)
        return math.log2(self.t) + 0.5 * math.log2(self.N) + 0.5 * math.log2((2.0 * self.N / 3.0 + 1.0) / 12.0)

    def predict(self, op, b_fresh):
        """op = (name, ch, n, budget, in0, in1, aux) -> predicted budget or None when the inputs are unknown"""
        name, _, n, _, in0, in1, aux = op
        if name == "Encryption":
            return self.fresh()[0]
        if in0 < 0:
            return None
        p0 = self.peak(in0)
        fresh_in = abs(in0 - b_fresh) <= 1  # a fresh ciphertext's noise is the uniform rounding term: peak = sqrt3 rms, not c rms
        shape = math.log2(self.c / math.sqrt(3.0)) if fresh_in else 0.0
        if name in ("Rotation", "ColumnRotation"):
            return self.budget(self.rss(p0, self.ks_gal))
        if name in ("Addition", "Subtraction"):
            if in1 < 0:
                return None
            return self.budget(self.rss(p0, self.peak(in1)))
        if name == "AddMany":
            if aux == 0:
                return None
            if aux > 0:  # scalar-MAC layer: aux = log2 rss of the weights of output 0 (>= 0); inputs are equally noisy
                return self.budget(p0 + aux + shape)
            return self.budget(aux)  # AddMany of ciphertexts: aux = log2 rss of the items' peaks (< 0)
        if name == "ScalarMultiplication":
            return self.budget(p0 + aux)
        if name == "PlainMultiplication":
            # a pair: the generic product (the noise polynomial is dense: gain (t/sqrt12) sqrt N) and the product of a Galois-invariant noise
            # (the output of a full SumAllSlots: one coefficient carries it, no sqrt N).  Partial slot sums lie in between.
            return (self.budget(p0 + self.plain_gain() + shape), self.budget(p0 + self.plain_gain() - 0.5 * math.log2(self.N)))
        if name in ("PlainAddition", "PlainSubtraction"):
            return in0
        if name == "Relinarization":
            if in1 < 0:
                return None
            m = self.mult_gain() + math.log2(2.0 ** p0 + 2.0 ** self.peak(in1))
            return self.budget(self.rss(m, self.ks_relin))
        return None


def render(recs, out):
    w = out.write
    w("# Per-operation noise budgets at the reference's parameters: measured by the GPU library (bit-exact, so independent of the GPU model) vs the analytic BFV model\n\n")
    w("Generated by `tools/noise_model.py` from the trace `tools/noise_trace.py` wrote on the GPU box (library option `trace_noise`:\n"
      "after every evaluator-level operation the invariant noise budget of its first output ciphertext is measured with the secret key,\n"
      "next to the budgets its inputs had).  `pred` is the model's output budget computed from the MEASURED input budgets of that one\n"
      "operation, so a deviation belongs to that operation alone.  Channel 0 (first plaintext modulus); `x n` = ciphertexts in the batched call.\n\n")
    summary = []
    worst_all = 0.0
    stats = {}
    for rec in recs:
        mdl = Model(rec, 0)
        bf, b_round, b_gauss = mdl.fresh()
        title = "%s, N=%d, k=%d (reference: %d, `%s`), m~ %s, %s weights" % (
            rec["topology"], rec["N"], rec["k"], rec["k_reference"], rec["reference"], "centred" if rec["mtilde_centered"] else "in [0,m~)", rec["weights"])
        w("## %s\n\n" % title)
        w("log2 q = %.1f, log2 t = %.1f; model: fresh %.1f (rounding term alone %.1f, Gaussian part alone %.1f), key switch floor %.1f (relin, w=%d) / %.1f (Galois, w=%d), "
          "dense multiply_plain costs %.1f bits, ct x ct %.1f bits + 1 (square)\n\n" % (
              mdl.logq, math.log2(mdl.t), bf, b_round, b_gauss, mdl.budget(mdl.ks_relin), rec["dbc"], mdl.budget(mdl.ks_gal), rec["dbc_galois"],
              mdl.plain_gain(), mdl.mult_gain()))
        w("| layer | operation | x n | in | measured | pred | diff |\n|---|---|---|---|---|---|---|\n")
        worst = 0.0
        mult_offsets = []
        for L in rec["layers"]:
            ops = [o for o in L["ops"] if o[1] == 0]
            # compress identical consecutive rows
            rows = []
            for o in ops:
                pred = mdl.predict(o, bf)
                name, _, n, b, in0, in1, aux = o
                ins = "-" if in0 < 0 else (str(in0) if in1 < 0 else "%d,%d" % (in0, in1))
                lo_hi = None
                if isinstance(pred, tuple):  # interval: inside it the deviation is zero, outside it the distance to the nearer end
                    lo_hi = pred
                    pred = min(max(b, pred[0]), pred[1]) if b > 3 else pred[0]
                diff = None if (pred is None or b <= 3 or min(x for x in (in0, in1) if x >= 0) <= 3 if (in0 >= 0 or in1 >= 0) else pred is None or b <= 3) else b - pred
                stats.setdefault(name + ("" if name != "Relinarization" else (", m~ centred" if rec["mtilde_centered"] else ", m~ in [0,m~)")), []).append(diff) if diff is not None else None
                if diff is not None and name == "Relinarization" and not rec["mtilde_centered"]:
                    mult_offsets.append(diff)
                    diff = None  # reported separately: the un-centred m~ convention adds a constant the centred model does not have
                if diff is not None:
                    worst = max(worst, abs(diff))
                key = (name, n, ins, b, None if pred is None else (round(pred, 1) if lo_hi is None else "%.1f..%.1f" % lo_hi))
                if rows and rows[-1][0] == key:
                    rows[-1][1] += 1
                else:
                    rows.append([key, 1, diff])
            for (name, n, ins, b, pred), rep, diff in rows:
                w("| %s | %s%s | %d | %s | %d | %s | %s |\n" % (L["layer"], name, "" if rep == 1 else " (x%d calls)" % rep, n, ins, b,
                                                             "-" if pred is None else (pred if isinstance(pred, str) else "%.1f" % pred),
                                                             "-" if diff is None else "%+.1f" % diff))
            w("| **%s** | layer output: budget %d..%d over %d ciphertexts, decrypts == Raw: **%s** | | | | | |\n" % (
                L["layer"], L["out_budget_min"], L["out_budget_max"], L["n_out_ct"], L["equals_raw"]))
        w("\nlargest |measured - pred| over the checked operations: **%.1f bits**" % worst)
        if mult_offsets:
            w("; ct x ct with m~ in [0,m~): measured - centred model = %s bits" % ", ".join("%+.1f" % x for x in mult_offsets))
        w("\n\n")
        worst_all = max(worst_all, worst)
        last = rec["layers"][-1]
        before = rec["layers"][-2]["out_budget_min"]
        summary.append((title, before, last["out_budget_min"], last["equals_raw"], worst))
    w("## Summary\n\n| run | budget entering the last layer | after it | scores == Raw | worst per-op deviation from the model |\n|---|---|---|---|---|\n")
    for t, b0, b1, eq, wd in summary:
        w("| %s | %d | %d | %s | %.1f |\n" % (t, b0, b1, eq, wd))
    w("\nworst deviation over all runs: %.1f bits\n" % worst_all)
    w("\n## Deviation by operation kind (measured - model, bits; operations with a budget <= 3 on either side are not scored: the measurement floors there)\n\n")
    w("| operation | scored | min | mean | max |\n|---|---|---|---|---|\n")
    for name in sorted(stats):
        d = stats[name]
        w("| %s | %d | %+.1f | %+.2f | %+.1f |\n" % (name, len(d), min(d), sum(d) / len(d), max(d)))
    w("\nNotes. `PlainMultiplication` is scored against the interval between the generic product (dense noise polynomial, gain (t/sqrt12) sqrt N) and the product of a "
      "Galois-invariant noise (the output of a full SumAllSlots, e.g. before the one-hot masks of ForceDenseFormat: one coefficient carries the noise and the sqrt N is "
      "absent).  `Relinarization` rows are multiply + relinearise; the centred model is shown for both m~ conventions, the un-centred one ([0,m~), the SEAL 3.2 reading) "
      "sits up to ~5 bits below it.\n")


if __name__ == "__main__":
    recs = json.load(open(sys.argv[1]))
    render(recs, sys.stdout)
