"""Square-activation micro-benchmark: multiply+relinearise of n ciphertexts through the raw ABI (N=8192, SEAL default q,
dbc=10), per-family device times.  Used for A/B runs of kernel variants (env knobs) and as the ncu target for those kernels.

--path fused|separate|both sets CNHE_MUL_FUSED (both: the two paths alternate in one process, `--rounds` times each).  For the fused
square it also times the size-3 product alone, where family 0 (ntt_forward) is exactly the fused kernel, and prints its kernel time,
FP64 issue share (DP instructions counted from the shapes) and HBM rate, with the card's name, power limit and maximum SM clock."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from cryptonets_b200.engine import Engine

ap = argparse.ArgumentParser()
ap.add_argument("n", type=int, nargs="?", default=256)
ap.add_argument("iters", type=int, nargs="?", default=5)
ap.add_argument("--path", choices=["fused", "separate", "both"], default="both")
ap.add_argument("--rounds", type=int, default=3)
args = ap.parse_args()
n, iters = args.n, args.iters

# H100 SXM FP64 issue ceiling, warp-level DP instructions per second (132 SMs x 2 per clock at 1.98 GHz)
DP_WARP_PEAK = 522.7e9


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().split("\n")[0]
        return [s.strip() for s in q.split(",")]
    except (OSError, subprocess.SubprocessError):
        return None


eng = Engine([549764251649], 8192, 10, 20)
eng.keygen(1)
eng.set_option("multi_stream", 0)
k, kt, N, logN = eng.k, eng.k + len(eng.bsk), 8192, 13
rng = np.random.default_rng(0)
q = np.array(eng.q, dtype=np.uint64)
host = (rng.integers(0, 1 << 62, (n, 2, k, N), dtype=np.uint64) % q[None, None, :, None]).astype(np.uint64)
a = eng.dev_from(host)
out = eng.dev_alloc(n * 2 * k * N)
out3 = eng.dev_alloc(n * 3 * k * N)
# per (ciphertext, residue): 5 N-point transforms (2 forward, 3 inverse) of N/2 log N butterflies at 8 DP instructions (fmodmul 6 + 2
# adds), the three products (3 fmodmul + 1 add per coefficient); re-centring and the last inverse stage's extra product are not counted
dp_warp = n * kt * (5 * (N // 2) * logN * 8 + 19 * N) / 32


def run(path):
    os.environ["CNHE_MUL_FUSED"] = "1" if path == "fused" else "0"
    for _ in range(2):
        eng.raw_multiply_relin(0, a, a, n, out)
    eng.sync()
    eng.prof_enable(True)
    t0 = time.perf_counter()
    eng.timer_start()
    for _ in range(iters):
        eng.raw_multiply_relin(0, a, a, n, out)
    host_ms = (time.perf_counter() - t0) * 1e3 / iters
    ms = eng.timer_stop_ms() / iters
    prof = eng.prof_collect()
    eng.prof_enable(False)
    res = {"path": path, "n": n, "ms": round(ms, 3), "host_issue_ms": round(host_ms, 3), "us_per_ct": round(ms * 1e3 / n, 2),
           "families_ms": {k_: round(v["ms"] / iters, 3) for k_, v in prof.items() if v["ms"] > 0}}
    if path == "fused":
        eng.raw_multiply(0, a, a, n, out3)
        eng.sync()
        eng.prof_enable(True)
        for _ in range(iters):
            eng.raw_multiply(0, a, a, n, out3)
        p3 = eng.prof_collect()
        eng.prof_enable(False)
        f = p3["ntt_forward"]
        kms = f["ms"] / iters
        res["square_fused"] = {"kernel_ms": round(kms, 3), "fp64_issue_share": round(dp_warp / DP_WARP_PEAK / (kms * 1e-3), 3),
                               "hbm_TBps": round(f["bytes"] / iters / (kms * 1e-3) / 1e12, 3),
                               "lift_floor_ms": round(p3["behz_elementwise"]["ms"] / iters, 3)}
    return res


c = card()
paths = ["fused", "separate"] if args.path == "both" else [args.path]
for r in range(args.rounds if args.path == "both" else 1):
    for path in paths:
        res = run(path)
        res["card"] = c
        print(json.dumps(res), flush=True)
