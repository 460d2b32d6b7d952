"""Operands that drive the FP64 path to the magnitudes its schedule guards against, and an exact integer model of that path.

The FP64 transforms keep residues lazy (DESIGN.md section 4): sums and differences are not reduced, fresh modular products come back
as a centred representative, and the host (`fp_schedule` in runtime.cu) re-centres only where the worst case could push an operand
of a modular product past 2^52.  Random operands stay far below that worst case (lazy values add up like a random walk), so these
builders construct the coherent cases instead: every value is an exact Python integer, every table comes from the CPU oracle.

No GPU is needed here.  tests/test_worst_case_inputs.py runs the model on these inputs; tests/test_gpu_worst_case_operands.py feeds
the same inputs to the kernels and compares with the oracle bit for bit."""
import numpy as np

TWO52 = 1 << 52
M_TILDE = 1 << 32
TARGET = 0.45  # fraction of p every constructed fresh product carries (its sign is known exactly below p/2)

# ---------------------------------------------------------------- the host schedule (port of fp_schedule, runtime.cu)
FWD_RADICES = {10: [2, 4, 4], 11: [3, 4, 4], 12: [4, 4, 4], 13: [5, 4, 4], 14: [5, 5, 4]}  # ntt_pass_radices(logN, 0)


def split_radices(logN):
    """passes of the split forward (CTA pairs at N = 16384, the fused kernels at 4096 / 8192)"""
    return [logN - 8, 4, 4]


def fp_schedule(p, logN):
    """the NttTab fields fp_schedule sets, computed with the same double arithmetic"""
    out = dict(fp_ok=0, fwd_recenter=0, inv_recenter=0, fwd_recenter_split=0, split_ok=0, split_out_rc=0, fwd_out_rc=0)
    if p.bit_length() > 49:
        return out
    L = 0.9 * 4503599627370496.0 / float(p)
    c = lambda a: 0.5 + 0.75 * a / (L / 0.9) + 1e-6

    def forward(rad):
        mask, A = 0, 1.0
        for i, r in enumerate(rad):
            for attempt in range(2):
                a = 0.51 if attempt else A
                ok = True
                for _ in range(r):
                    ok = ok and a < L
                    a += c(a)
                ok = ok and a < L
                if ok:
                    A = a
                    if attempt:
                        mask |= 1 << i
                    break
                if attempt or i == 0:
                    return None
        return mask, A

    f = forward(FWD_RADICES[logN])
    if f is None:
        return out
    out["fwd_recenter"], A = f
    out_rc = lambda a: int(a * a * float(p) >= 0.9 * 2251799813685248.0)
    if logN >= 12:
        s = forward(split_radices(logN))
        out["split_ok"] = int(s is not None)
        if logN == 14:
            if s is None:
                return out
            out["fwd_recenter_split"] = s[0]
            A = max(A, s[1])
        elif s is not None:
            out["fwd_recenter_split"] = s[0]
            out["split_out_rc"] = out_rc(s[1])
    out["fwd_out_rc"] = out_rc(A)
    A = 1.25
    for v in range(logN):
        if 2 * A >= L:
            return out
        y = c(2 * A)
        x = 2 * A
        if 2 * x >= L:
            out["inv_recenter"] |= 1 << v
            x = 0.51
        A = max(x, y)
    if A >= L:
        return out
    out["fp_ok"] = 1
    return out


# ---------------------------------------------------------------- exact model of the lazy FP64 networks
def centred(x, p):
    """centred representative in (-p/2, p/2] of integers (Python int or object array): what frecenter / fmodmul return"""
    r = x % p
    return np.where(r > p // 2, r - p, r) if isinstance(r, np.ndarray) else (r - p if r > p // 2 else r)


def _amax(x):
    return int(np.abs(x).max())


def _obj(a):
    return np.array([int(v) for v in np.asarray(a).ravel()], dtype=object)


def centred_table(w, p):
    return _obj([centred(int(v), p) for v in w])


def lazy_forward(a, p, wd, rad, mask):
    """CT network of k_ntt_forward_fp / the split kernels on input a (canonical or lazy integers): sums and differences exact,
    products centred, every value of pass i re-centred first where bit i of mask is set.  Returns (lazy output, peak |value|)."""
    x = _obj(a)
    N = len(x)
    peak = _amax(x)
    s = 0
    for i, r in enumerate(rad):
        if (mask >> i) & 1:
            x = centred(x, p)
        for _ in range(r):
            gap = N >> (s + 1)
            v = x.reshape(1 << s, 2, gap)
            t = centred(v[:, 1, :] * wd[1 << s: 2 << s].reshape(-1, 1), p)
            x = np.stack([v[:, 0, :] + t, v[:, 0, :] - t], axis=1).reshape(N)
            peak = max(peak, _amax(x))
            s += 1
    return x, peak


def lazy_inverse(a, p, iwd, inv_n, mask):
    """GS network of the FP64 inverse: sums exact, differences times the twiddle centred, the sums of stage v re-centred where bit v
    of mask is set; the last stage folds N^-1 into both products.  Returns (lazy output, peak |value|)."""
    x = _obj(a)
    N = len(x)
    logN = N.bit_length() - 1
    peak = _amax(x)
    n_w = centred(inv_n * int(iwd[1]), p)
    for v in range(logN):
        h = 1 << v
        y = x.reshape(N >> (v + 1), 2, h)
        s, d = y[:, 0, :] + y[:, 1, :], y[:, 0, :] - y[:, 1, :]
        peak = max(peak, _amax(s), _amax(d))
        if v == logN - 1:
            s, d = centred(s * centred(inv_n, p), p), centred(d * n_w, p)
        else:
            d = centred(d * iwd[(N >> (v + 1)): (N >> v)].reshape(-1, 1), p)
            if (mask >> v) & 1:
                s = centred(s, p)
        x = np.stack([s, d], axis=1).reshape(N)
    return x, peak


# ---------------------------------------------------------------- forward (CT) worst case
def forward_path_targets(N):
    """outputs whose paths are built: both ends and the half boundary of the split kernels"""
    return [0, N // 2 - 1, N // 2, N - 1]


def _solve(w, p, sign, limit=None):
    """y in [0, limit) whose centred product with w is nearest sign * TARGET * p (exactly that class when limit is None)"""
    goal = sign * int(TARGET * p)
    if limit is None or limit >= p:
        return goal * pow(w, -1, p) % p
    if limit > 1 << 16 and limit < p >> 16:
        return _near_class(w, p, goal, limit)
    if limit > 1 << 16:  # walk the classes outwards from the goal until one has a small enough preimage
        wi = pow(w, -1, p)
        for off in range(1 << 20):
            for t in (goal - off, goal + off):
                if t * wi % p < limit:
                    return t * wi % p
    ys = np.arange(limit, dtype=object)
    prods = centred(ys * w, p)
    return int(ys[int(np.argmin([abs(int(v) - goal) for v in prods]))])


def _near_class(w, p, goal, limit):
    """y in [0, limit) whose centred product with w is near goal, for preimage ranges too sparse to walk (limit / p below 2^-16): the
    lattice {(s y, w y + p z)}, s = p // limit, weighs both coordinates alike; Babai rounding on its Lagrange-reduced basis gives a
    vector near (s limit / 2, goal), so y is near limit / 2 and the product within about p / sqrt(limit) of goal"""
    from fractions import Fraction
    s = max(1, p // limit)
    b1, b2 = (s, w % p), (0, p)
    n2 = lambda v: v[0] * v[0] + v[1] * v[1]
    if n2(b1) > n2(b2):
        b1, b2 = b2, b1
    while True:
        mu = round(Fraction(b1[0] * b2[0] + b1[1] * b2[1], n2(b1)))
        b2 = (b2[0] - mu * b1[0], b2[1] - mu * b1[1])
        if n2(b2) >= n2(b1):
            break
        b1, b2 = b2, b1
    tx, ty = s * (limit // 2), goal
    det = b1[0] * b2[1] - b1[1] * b2[0]
    c1, c2 = Fraction(tx * b2[1] - ty * b2[0], det), Fraction(b1[0] * ty - b1[1] * tx, det)
    best = None
    for d1 in (-1, 0, 1, 2):
        for d2 in (-1, 0, 1, 2):
            a1, a2 = c1.__floor__() + d1, c2.__floor__() + d2
            y = (a1 * b1[0] + a2 * b2[0]) // s
            if 0 <= y < limit:
                err = abs(centred(w * y, p) - goal)
                if best is None or err < best[0]:
                    best = (err, y)
    if best is None:
        raise ValueError("no preimage below %d" % limit)
    return best[1]


def forward_worst_case(p, wd, out_index, digit_bits=None, negative=False, limit=None):
    """Canonical input whose lazy value on the path from input 0 to output `out_index` grows by TARGET*p at every stage.

    a[0] is maximal.  On that path the path value is always the upper operand of its butterfly; the partner at stage s is input
    N >> (s+1) on its own (its subtree holds nothing else), so one coefficient per stage is solved to make w*y = +-TARGET p, with the
    sign that adds to the path on the branch the output takes.  digit_bits: every coefficient below 2^digit_bits (a digit plane);
    limit: every coefficient below limit (<= p) instead.  negative: every product subtracts instead, so the output ends near
    -(logN TARGET - 1) p."""
    N = len(wd)
    logN = N.bit_length() - 1
    if limit is None:
        limit = None if digit_bits is None else min(1 << digit_bits, p)
    a = [0] * N
    a[0] = (p - 1) if limit is None else limit - 1
    pos = 0
    for s in range(logN):
        gap = N >> (s + 1)
        lower = (out_index >> (logN - 1 - s)) & 1
        w = int(wd[(1 << s) + (pos >> (logN - s))]) % p
        a[gap] = _solve(w, p, (-1 if lower else 1) * (-1 if negative else 1), limit)
        pos += gap * lower
    return np.array(a, dtype=np.uint64)


def forward_path_sum(p, logN, digit_bits=None):
    """the path's analytic largest magnitude with no re-centre: maximal input plus a product of p/2 at every stage"""
    top = (p - 1) if digit_bits is None else min(1 << digit_bits, p) - 1
    return top + logN * (p // 2)


# ---------------------------------------------------------------- inverse (GS) worst case
def constant_class(p, sign=1):
    """lazy NTT-domain value of the constant class: sign * TARGET * p, centred"""
    return sign * int(TARGET * p)


def inverse_constant(p, after_stage=-1):
    """Canonical constant c (an NTT-domain constant: its inverse is c * delta_0) whose coefficient-0 sums are largest in the segment
    after the re-centre of stage `after_stage`: the sums of stage v are 2^(v+1) c, so a re-centre there leaves
    centred(2^(after_stage+1) c), made TARGET p here.  after_stage = -1: the first segment, c = p - 1."""
    if after_stage < 0:
        return p - 1
    return int(TARGET * p) * pow(2, -(after_stage + 1), p) % p


def inverse_segments(mask, logN):
    """(stage of the re-centre, stage of the re-centre before it or -1) for every bit of an inverse schedule that a kernel applies:
    the sums of the last stage are multiplied by N^-1 at once, so a bit there has nothing to re-centre"""
    bits = [b for b in range(logN - 1) if (mask >> b) & 1]
    return [(b, bits[i - 1] if i else -1) for i, b in enumerate(bits)]


def square_root_near_target(p, seed=0):
    """v with v^2 = +-TARGET p (mod p) up to 1 %: the impulse v * delta_0 transforms to the constant v, squares to the constant v^2"""
    rng = np.random.default_rng(seed + p % 1000003)
    lo, hi = int((TARGET - 0.01) * p), int(TARGET * p)
    while True:
        v = int(rng.integers(1, p - 1))
        r = abs(centred(v * v, p))
        if lo <= r <= hi:
            return v


def key_constant(p, v):
    """K with K*v = TARGET p (mod p): the NTT-domain key word that turns the digit constant v into the worst product"""
    return int(TARGET * p) * pow(v % p, -1, p) % p


# ---------------------------------------------------------------- NTT-friendly primes of a chosen width
def is_prime(n):
    if n < 2:
        return False
    for sp in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):
        if n % sp == 0:
            return n == sp
    d, s = n - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    for a in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):  # deterministic below 3.3e24
        x = pow(a, d, n)
        if x in (1, n - 1):
            continue
        for _ in range(s - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def primes(bits, N, count=1):
    """the `count` largest `bits`-bit primes = 1 mod 2N, descending (none of them 48-bit, so none is a fast Bsk prime)"""
    assert bits != 48
    out, c = [], ((1 << bits) - 1) // (2 * N) * (2 * N) + 1
    while len(out) < count:
        if is_prime(c):
            out.append(c)
        c -= 2 * N
    assert all(p.bit_length() == bits for p in out)
    return out


GAMMA = 0x1fffffffffc80001  # the decryption's auxiliary prime (SEAL small_mods)
M_SK = 0x1fffffffffe00001   # SEAL's m_sk; SEAL's auxiliary base primes are the next 61-bit primes = 1 mod 2^18


def clear_primes(bits, N, count=1):
    """the `count` largest `bits`-bit primes = 1 mod 2N that are neither gamma, nor m_sk, nor = 1 mod 2^18 (so no SEAL auxiliary base
    prime at any k): coefficient moduli every context and the oracle accept"""
    assert bits != 48
    out, c = [], ((1 << bits) - 1) // (2 * N) * (2 * N) + 1
    while len(out) < count:
        if (c - 1) % (1 << 18) and is_prime(c):
            out.append(c)
        c -= 2 * N
    assert all(p.bit_length() == bits for p in out) and GAMMA not in out and M_SK not in out
    return out


# ---------------------------------------------------------------- decryption on big integers (no gamma, no oracle)
def ternary_secret(sk_coeff, q):
    """the secret key's coefficients in {-1, 0, 1} from its residues [k][N] in coefficient form; every residue must say the same"""
    sk = np.asarray(sk_coeff, np.uint64).reshape(len(q), -1)
    s = np.where(sk[0] == 1, 1, np.where(sk[0] == q[0] - 1, -1, 0)).astype(np.int64)
    for l, p in enumerate(q):
        assert np.array_equal(sk[l], np.where(s < 0, p - 1, s).astype(np.uint64)), "not one ternary polynomial"
    return s


def _kron(a):
    """Kronecker substitution: coefficients below 2^64 as one integer, 128 bits apart"""
    w = np.zeros((len(a), 2), np.uint64)
    w[:, 0] = a
    return int.from_bytes(w.tobytes(), "little")


def _unkron(x, n):
    w = np.frombuffer(x.to_bytes(16 * n, "little"), np.uint64).reshape(n, 2)
    return w[:, 0].astype(object) + (w[:, 1].astype(object) << 64)


def times_ternary(c, s, p):
    """c(x) s(x) mod (x^N + 1, p), c in [0, p)^N, s in {-1, 0, 1}^N, exactly (every product coefficient stays below 2^128)"""
    N = len(c)
    C = _kron(np.asarray(c, np.uint64))
    full = _unkron(C * _kron((s == 1).astype(np.uint64)), 2 * N) - _unkron(C * _kron((s == -1).astype(np.uint64)), 2 * N)
    return (full[:N] - full[N:]) % p


def exact_decrypt(ct, s, q, t):
    """the plaintext round(t [c0 + c1 s]_Q / Q) mod t of a size-2 ciphertext [2][k][N] (coefficient form), on Python integers"""
    k = len(q)
    ct = np.asarray(ct, np.uint64).reshape(2, k, -1)
    Q = 1
    for p in q:
        Q *= p
    x = 0
    for l, p in enumerate(q):
        r = (ct[0, l].astype(object) + times_ternary(ct[1, l], s, p)) % p
        x = x + r * ((Q // p) * pow(Q // p % p, -1, p))
    x = x % Q
    return ((2 * t * x + Q) // (2 * Q) % t).astype(np.uint64)


# ---------------------------------------------------------------- digit decomposition (make_digit_map, runtime.cu)
def digit_map(q, w):
    """[(residue index, shift)] in digit order; more than 64 digits is refused"""
    dm = [(i, s) for i, qi in enumerate(q) for s in range(0, qi.bit_length(), w)]
    if len(dm) > 64:
        raise ValueError("decomposition bit count too small: more than 64 digits")
    return dm


def digit_worst_case_target(q, w, wd_of, out_index):
    """c2 residues (k x N) whose every digit plane is the forward worst case of its digit under modulus d % k.
    wd_of(l): centred forward twiddles of q_l.  Words stay below q_i (the top digit is bounded by q_i's top bits)."""
    k, N = len(q), len(wd_of(0))
    words = [[0] * N for _ in range(k)]
    for d, (i, sh) in enumerate(digit_map(q, w)):
        l = d % k
        bits = min(w, q[i].bit_length() - sh)
        plane = forward_worst_case(q[l], wd_of(l), out_index, bits)
        for j in range(N):
            words[i][j] |= int(plane[j]) << sh
    for i in range(k):
        for j in range(N):
            if words[i][j] >= q[i]:
                words[i][j] %= q[i]
    return np.array(words, dtype=np.uint64)


# ---------------------------------------------------------------- BEHZ extremes
def mont_rq_r(x, q):
    """r of fastbconv_mtilde + mont_rq for the coefficient whose CRT value is x (k_behz_lift, behz.cu)"""
    Q = 1
    for qi in q:
        Q *= qi
    s = 0
    for qi in q:
        qhat = Q // qi
        tmp = (x % qi) * (M_TILDE % qi) % qi * pow(qhat % qi, -1, qi) % qi
        s += tmp * (qhat % M_TILDE)
    s %= M_TILDE
    return (M_TILDE - s * pow(Q % M_TILDE, -1, M_TILDE) % M_TILDE) % M_TILDE


def mont_rq_word(q, r_target, seed=0):
    """CRT value x in [0, Q) with mont_rq_r(x) == r_target.  r = floor(m~ x / Q) - u (mod m~), u < k the overflow count of the
    fast base conversion: for each u, search the interval of x where floor(m~ x / Q) = r + u."""
    Q = 1
    for qi in q:
        Q *= qi
    rng = np.random.default_rng(seed)
    for f in [r_target + u for u in range(len(q))] + [r_target - M_TILDE + u for u in range(len(q))]:
        if not 0 <= f < M_TILDE:
            continue
        lo, hi = -(-f * Q // M_TILDE), ((f + 1) * Q - 1) // M_TILDE
        if hi < lo:
            continue
        cands = [lo, hi, (lo + hi) // 2] + [lo + int(rng.integers(0, 1 << 62)) * (hi - lo) // (1 << 62) for _ in range(200)]
        for x in cands:
            if 0 <= x < Q and mont_rq_r(x, q) == r_target:
                return x
    raise ValueError("no word found for r = %d" % r_target)


def residues(x, q):
    return [x % qi for qi in q]


def behz_extreme_cts(q, N, fresh):
    """ciphertexts (2 x k x N words each) at the BEHZ bounds: all (q_i - 1), all zero, c0 maximal with c1 zero, and a fresh ciphertext
    carrying the mont_rq words r = 2^31 - 1, 2^31 (the centred-m~ tie) and 2^32 - 1 at both ends of both polynomials"""
    k = len(q)
    top = np.array(q, dtype=np.uint64)[:, None] - np.uint64(1)
    full = np.broadcast_to(top, (k, N))
    zero = np.zeros((k, N), np.uint64)
    out = [np.stack([full, full]), np.stack([zero, zero]), np.stack([full, zero])]
    ct = np.array(fresh, dtype=np.uint64).reshape(2, k, N).copy()
    for n, r in enumerate((M_TILDE // 2 - 1, M_TILDE // 2, M_TILDE - 1)):
        x = mont_rq_word(q, r, seed=n)
        for part in range(2):
            for j in (n, N - 1 - n):
                ct[part, :, j] = residues(x, q)
    out.append(ct)
    return [c.reshape(-1).copy() for c in out]


# ---------------------------------------------------------------- closed-form key switch
def key_switch_reference(orc, target, keys, dbc, planes=None):
    """(2 x k x N) INTT(sum_d NTT(digit_d) * K_d) mod q_l for target residues (k x N) and NTT-domain keys (D x 2 x k x N), from the
    oracle's transforms: the part a key switch adds to its base.  planes: signed integer digit planes (D x N) in place of the digits
    of a target (the plane-source key switch; target is then unused), taken modulo each q_l."""
    q, N = orc.q, orc.N
    k = len(q)
    dm = digit_map(q, dbc)
    keys = np.asarray(keys, dtype=np.uint64).reshape(len(dm), 2, k, N)
    out = np.zeros((2, k, N), np.uint64)
    if planes is not None:
        planes = np.asarray(planes, dtype=np.int64).reshape(len(dm), N)
    for l in range(k):
        ql = q[l]
        if planes is not None:
            digits = (planes % ql).astype(np.uint64)  # numpy's % takes the divisor's sign: canonical residues
        else:
            digits = np.stack([((np.asarray(target[i], dtype=np.uint64) >> np.uint64(sh)) & np.uint64((1 << dbc) - 1)).astype(object) % ql
                               for i, sh in dm]).astype(np.uint64)
        nt = orc.ntt_batch(l, digits).astype(object)
        for part in range(2):
            acc = (nt * keys[:, part, l, :].astype(object)).sum(axis=0) % ql
            out[part, l] = orc.ntt(l, acc.astype(np.uint64), inverse=True)
    return out


def add_mod(a, b, q):
    k = len(q)
    qa = np.array(q, dtype=object).reshape((1,) * (np.ndim(a) - 2) + (k, 1))
    return ((np.asarray(a).astype(object) + np.asarray(b).astype(object)) % qa).astype(np.uint64)


def behz_lift(x, q, centred):
    """the integer k_behz_lift carries into the auxiliary base for the coefficient whose CRT value is x: x + c Q, c in {0, 1}
    (or c in {-1, 0} with the centred m~)"""
    Q = 1
    for qi in q:
        Q *= qi
    S = sum((x % qi) * (M_TILDE % qi) % qi * pow((Q // qi) % qi, -1, qi) % qi * (Q // qi) for qi in q)
    r = mont_rq_r(x, q)
    rr = r - M_TILDE if centred and r >= M_TILDE // 2 else r
    return (S + Q * rr) // M_TILDE


def bsk_forward_worst_ct(q, b, wd_b, out_index, centred):
    """Ciphertext whose coefficients lift to the integers of forward_worst_case under the auxiliary prime b, positive in c0 and
    negative in c1: the forward transform of that residue inside the multiply reaches its bound, and the square multiplies two lazy
    outputs of opposite sign at their bound (c0 c1), whose quotient is the one the FP64 product cannot round past -2^51."""
    Q = 1
    for qi in q:
        Q *= qi
    k, N = len(q), len(wd_b)
    ct = np.zeros((2, k, N), np.uint64)
    for part in range(2):
        ct[part] = _lifting_to(q, Q, b, forward_worst_case(b, wd_b, out_index, negative=part == 1), centred)
    return ct.reshape(-1)


def _lifting_to(q, Q, b, targets, centred):
    """residues (k x N) of words whose BEHZ lift is congruent to targets modulo b"""
    xs = []
    for t in (int(v) for v in targets):
        x = t
        for _ in range(8):
            lifted = behz_lift(x, q, centred)
            if lifted % b == t:
                break
            x = (t - (lifted - x)) % b  # cancel the c Q the lift added
        else:
            raise ValueError("no word lifts to %d" % t)
        xs.append(x)
    return np.array([[x % qi for x in xs] for qi in q], dtype=np.uint64)
