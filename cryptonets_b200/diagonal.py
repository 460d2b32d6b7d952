"""Exact (mod t) numpy model of the diagonal matrix-vector product with baby-step / giant-step (cnhe_mat_mul_diagonal, DESIGN.md
section 4.10), on a ciphertext's slot semantics: N slots as two rows of N/2, rotate_rows(s) moves column x + s of both rows to column x,
rotate_columns swaps the rows.  It also restates the library's choice of the number of baby steps n1, so that both can be checked without
a GPU.  The folded product for matrices with few rows (cnhe_diag_prepare_folded) is modelled the same way, with its planner."""
import numpy as np


def rotate_rows(v, s):
    """Slot vector after rotate_rows(s): slot (a, x) takes the value of slot (a, x + s mod N/2)."""
    half = len(v) // 2
    r = np.asarray(v).reshape(2, half)
    return np.roll(r, -s, axis=1).reshape(-1)


def rotate_columns(v):
    half = len(v) // 2
    return np.asarray(v).reshape(2, half)[::-1].reshape(-1)


def standard_galois_elts(N):
    """The Galois elements a context generates keys for: 2N - 1 (rotate_columns), then 3^(2^i) and 3^(-2^i) mod 2N."""
    m = 2 * N
    out, p3, n3 = [m - 1], 3, pow(3, -1, m)
    for _ in range(N.bit_length() - 2):
        out += [p3, n3]
        p3, n3 = p3 * p3 % m, n3 * n3 % m
    return out


def rotation_hops(N, galois_elts):
    """hops[s]: key switches of rotate_rows(s), 0 <= s < N/2 -- one with the step's own key, else one per term of its non-adjacent form
    (a term of N/2 is the identity and skipped)."""
    half, m, elts = N // 2, 2 * N, set(int(e) for e in galois_elts)
    hops = [0] * half
    for s in range(1, half):
        if pow(3, s, m) in elts:
            hops[s] = 1
            continue
        v, i = s, 0
        while v:
            z = (2 - (v & 3)) if v & 1 else 0
            v = (v - z) >> 1
            if z and (1 << i) != half:
                hops[s] += 1
            i += 1
    return hops


def diagonal_flags(M, N):
    """nz[b, s]: whether generalised diagonal (b, s) of M (R x dim, R, dim <= N) has a nonzero weight."""
    half = N // 2
    R, dim = M.shape
    nz = np.zeros((2, half), bool)
    rows = np.arange(R)
    a, x = rows // half, rows % half
    for b in range(2):
        for s in range(half):
            col = (a ^ b) * half + (x + s) % half
            ok = col < dim
            nz[b, s] = np.any(M[rows[ok], col[ok]] != 0)
    return nz


def key_switch_cost(nz, hops, n1):
    """Key switches per input vector with n1 baby steps (what the library minimises)."""
    half = len(hops)
    baby = np.zeros((2, n1), bool)
    giant = np.zeros(half // n1, bool)
    for b, s in zip(*np.nonzero(nz)):
        baby[b, s % n1] = True
        giant[s // n1] = True
    cost = sum(hops[h] for b in range(2) for h in range(n1) if baby[b, h])
    cost += 1 if baby[1].any() else 0
    cost += sum(hops[n1 * g] for g in range(1, half // n1) if giant[g])
    return cost


def plan_baby_steps(nz, N, galois_elts):
    """The library's n1: the power of two dividing N/2 with the fewest key switches, the smallest on a tie."""
    hops = rotation_hops(N, galois_elts)
    cands = [1 << i for i in range((N // 2).bit_length())]
    costs = {n1: key_switch_cost(nz, hops, n1) for n1 in cands}
    return min(cands, key=lambda n1: (costs[n1], n1)), costs


def prerotated_diagonals(M, N, n1, t):
    """{(b, g, h): slot vector} of the nonzero diagonals, diagonal (b, n1 g + h) rotated right by n1 g, mod t (what cnhe_diag_prepare
    encodes)."""
    half = N // 2
    R, dim = M.shape
    assert t < 2 ** 31  # products of two residues stay exact in int64
    Mt = np.zeros((N, N), dtype=np.int64)
    Mt[:R, :dim] = np.asarray(M, dtype=np.int64) % t
    nz = diagonal_flags(np.asarray(M, dtype=np.int64) % t, N)
    i = np.arange(N)
    a, x = i // half, i % half
    out = {}
    for g in range(half // n1):
        for b in range(2):
            for h in range(n1):
                if not nz[b, g * n1 + h]:
                    continue
                row = a * half + (x - n1 * g) % half
                col = (a ^ b) * half + (x + h) % half
                out[(b, g, h)] = Mt[row, col]
    return out


def product(diags, v, N, n1, t):
    """y = sum_g rotate_rows(n1 g)( sum_{b,h} D'[b,g,h] * rotate_columns^b rotate_rows(h)(v) ) mod t, with v zero-padded to N slots."""
    vv = np.zeros(N, dtype=np.int64)
    vv[:len(v)] = np.asarray(v, dtype=np.int64) % t
    baby = {(0, h): rotate_rows(vv, h) for h in range(n1)}
    kv = rotate_columns(vv)
    baby.update({(1, h): rotate_rows(kv, h) for h in range(n1)})
    inner = {}
    for (b, g, h), d in diags.items():
        inner[g] = (inner.get(g, 0) + d * baby[(b, h)]) % t
    y = np.zeros(N, dtype=np.int64)
    for g, acc in inner.items():
        y = (y + rotate_rows(acc, n1 * g)) % t
    return y


def folded_flags(M, N):
    """nz[d], d < N/2: whether some nonzero weight M[r, col] has col - r = d mod N/2 (what the prepare's flags pass marks).  Wrapped
    diagonal j of fold width W is nonzero exactly when nz[d] holds for some d = j mod W."""
    half = N // 2
    r, col = np.nonzero(np.asarray(M))
    nz = np.zeros(half, bool)
    nz[(col - r) % half] = True
    return nz


def wrapped_flags(nz, W):
    """[2][N/2] flags in key_switch_cost's layout (b = 0 only) of the wrapped diagonals of fold width W."""
    half = len(nz)
    out = np.zeros((2, half), bool)
    for d in np.nonzero(nz)[0]:
        out[0, d % W] = True
    return out


def folded_cost(nz, hops, W, n1, dim):
    """Key switches per input of the folded product: the BSGS rotations, the column fold when dim > N/2, and log2(N/2 / W) row folds."""
    half = len(hops)
    return key_switch_cost(wrapped_flags(nz, W), hops, n1) + (1 if dim > half else 0) + (half // W).bit_length() - 1


def plan_folded(M, N, galois_elts, fold_width=0, baby_steps=0):
    """The library's (W, n1, key switches): the fewest key switches over the powers of two R <= W <= N/2 (or the given W) and n1 dividing
    W (or the given n1); on a tie the smaller W, then the smaller n1."""
    half = N // 2
    R, dim = np.asarray(M).shape
    nz = folded_flags(M, N)
    hops = rotation_hops(N, galois_elts)
    ws = [fold_width] if fold_width else [w for w in (1 << i for i in range(half.bit_length())) if R <= w <= half]
    best = None
    for W in ws:
        for n1 in ([baby_steps] if baby_steps else [1 << i for i in range(W.bit_length())]):
            if n1 > W:
                continue
            cost = folded_cost(nz, hops, W, n1, dim)
            if best is None or cost < best[2]:
                best = (W, n1, cost)
    return best


def folded_diagonals(M, N, W, n1, t):
    """{(0, g, h): slot vector} of the nonzero wrapped diagonals E_{n1 g + h}[(a, x)] = M[x mod W, a N/2 + (x + n1 g + h mod N/2)], each
    rotated right by n1 g, mod t (what cnhe_diag_prepare_folded encodes)."""
    half = N // 2
    M = np.asarray(M, dtype=np.int64) % t
    R, dim = M.shape
    Mt = np.zeros((half, N), dtype=np.int64)
    Mt[:R, :dim] = M
    nz = wrapped_flags(folded_flags(M, N), W)[0]
    i = np.arange(N)
    a, x = i // half, i % half
    out = {}
    for j in range(W):
        if nz[j]:
            g, h = divmod(j, n1)
            out[(0, g, h)] = Mt[(x - n1 * g) % W, a * half + (x + h) % half]
    return out


def folded_product(diags, v, N, W, n1, R, dim, t):
    """The folded product: the BSGS sum over the stored diagonals, the column fold when dim > N/2, the row folds by W, 2W, ..., N/4 and the
    mask of slots 0 .. R - 1, mod t."""
    half = N // 2
    y = product(diags, v, N, n1, t)
    if dim > half:
        y = (y + rotate_columns(y)) % t
    s = W
    while s < half:
        y = (y + rotate_rows(y, s)) % t
        s *= 2
    y[R:] = 0
    return y
