"""Python restatement of how doubles enter and leave the plaintext channels (DESIGN 4.19), with Python integers: the split of a value into
residues (the wrapper's SplitBigNumbers) and the centred CRT join of residues back into a double (JoinSplitNumbers).  Python's float
product, round() and float(int) are IEEE round-to-nearest-even, so the join's doubles compare bit for bit with the library's."""
import math

LIMIT = 1.5e38


def big_factor(ts):
    return math.prod(int(t) for t in ts)


def crt_coeffs(ts):
    """coefficient i: (B / t_i) ((B / t_i)^-1 mod t_i), below B"""
    B = big_factor(ts)
    return [(B // int(t)) * pow((B // int(t)) % int(t), -1, int(t)) % B for t in ts]


def split_value(v, scale, ts):
    """The residues of one value: w = rint(v scale) (ties to even); None when |w| >= 1.5e38 or v scale is not finite."""
    x = float(v) * float(scale)
    if not math.isfinite(x):
        return None
    w = round(x)
    if not abs(w) < LIMIT:
        return None
    B = big_factor(ts)
    mag = abs(w)
    if mag >= B:
        mag %= B
    z = B - mag if (w < 0 and mag) else mag
    return [z % int(t) for t in ts]


def split(values, scale, ts):
    """[P][len(values)] residues of a flat sequence of values; ValueError when one is out of range."""
    out = [[] for _ in ts]
    for v in values:
        r = split_value(v, scale, ts)
        if r is None:
            raise ValueError("value out of range")
        for i, x in enumerate(r):
            out[i].append(x)
    return out


def join_value(residues, scale, ts):
    """The double of one value's residues: the CRT sum mod B, centred (2 acc > B -> -(B - acc)), over scale."""
    B = big_factor(ts)
    acc = sum(c * int(r) for c, r in zip(crt_coeffs(ts), residues)) % B
    val = -float(B - acc) if acc * 2 > B else float(acc)
    return val / float(scale)


def join(residues, scale, ts):
    """residues [P][n] -> n doubles"""
    return [join_value([residues[i][j] for i in range(len(ts))], scale, ts) for j in range(len(residues[0]))]
