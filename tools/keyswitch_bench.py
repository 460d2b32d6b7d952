"""Key-switch micro-benchmark: relinearisation of n size-3 ciphertexts through the raw ABI (N=8192, SEAL default q, dbc=10, one
stream), per-family device times and the HBM bytes the two key-switch forms need, computed from the shapes.

    python tools/keyswitch_bench.py [n ...] [--iters I] [--path auto|fused|digits]

During a relinearise-only call on the digit path family 0 (ntt_forward) is the digit transforms, family 3 (keyswitch_mac) the key
product and family 1 (ntt_inverse) the inverse transforms with the base addition.  On the fused path family 3 is the one kernel that
does all three, and families 0 and 1 stay empty.  `--path` sets CNHE_KS_FUSED for the run (auto: the library's own choice by n).  One
JSON line per n.

The fused kernel's operands come from L2: every (ciphertext, residue, half) CTA reads both halves of the source residue (8N bytes) and
its half of the two key polynomials (8N bytes as u64 words, 6N in the 48-bit packed copy the library uses while every q_l < 2^48) per
digit.  The line reports those bytes for both key forms and the achieved rate against --l2-tbs, the L2 read bandwidth tools/l2_bench
measures (7.4 TB/s on one H100 80GB HBM3 at 700 W, 32 MiB buffer)."""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

ap = argparse.ArgumentParser()
ap.add_argument("n", type=int, nargs="*", default=[1, 8, 32, 64, 128, 945])
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--path", choices=["auto", "fused", "digits"], default="auto")
ap.add_argument("--l2-tbs", type=float, default=7.4, help="L2 read bandwidth to compare the fused kernel's rate with (tools/l2_bench)")
args = ap.parse_args()
if args.path != "auto":
    os.environ["CNHE_KS_FUSED"] = "1" if args.path == "fused" else "0"

from cryptonets_b200.engine import Engine

eng = Engine([549764251649], 8192, 10, 20)
eng.keygen(1)
eng.set_option("multi_stream", 0)
k, N = eng.k, 8192
D = sum((int(q).bit_length() + 9) // 10 for q in eng.q)  # base-2^10 digits of every residue
q = np.array(eng.q, dtype=np.uint64)
packed = max(eng.q) < 1 << 48
rng = np.random.default_rng(0)
# FP64 instructions per thread of a (ciphertext, residue, half) CTA of the fused kernel at N = 8192 (4096-point halves, 256 threads, 16
# coefficients each).  Per digit: stage 0 folded into the loads (16 modular products + 16 adds), 12 radix-2 stages of 8 butterflies
# (6 + 2), the key product (32 modular products + 32 adds), digit conversions (32 u2d) and key conversions (32 u2d).  Once per CTA, the
# epilogue's inverse of both key polynomials: 12 in-half stages of 8 butterflies each, then the cross-half stage (16 adds and modular
# products by N^-1) and 16 conversions to integers
FMODMUL, BFLY = 6, 8
DP_PER_THREAD = 16 * (FMODMUL + 1) + 12 * 8 * BFLY + 32 * (FMODMUL + 1) + 32 + 32
DP_INVERSE_PER_THREAD = 2 * (12 * 8 * BFLY + 16 * (FMODMUL + 1) + 16)
DP_WARP_INSTR_PER_CT = (DP_PER_THREAD * D + DP_INVERSE_PER_THREAD) * (256 // 32) * 2 * k


def l1_wavefronts_per_cta_digit(key_word, grouped):
    """128-byte L1 / shared-memory data-path wavefronts of one CTA and one digit (N = 8192: 4096-point half, 256 threads, 8 warps),
    counted from the shapes: work buffer (pass-1 store, pass-2 load + store, last-pass load), the polynomial-1 accumulator (load +
    store; polynomial 0's sits in registers), twiddle-cache reads of passes 1-2 (15 distinct words per thread and pass, one wavefront per warp load), source words (both
    halves, coalesced), key words (two polynomials, coalesced) and the last pass's 15 twiddles per thread: 8 warp loads of 512
    contiguous bytes from the grouped table, or scalar loads whose lanes sit 2^u words apart at stage u (a warp load touches
    min(32, 2^(u+1)) lines, 2^u loads per stage).  A model: not measured."""
    H, T, W = 4096, 256, 8
    work = 4 * H * 8 // 128
    acc = 2 * H * 8 // 128
    twc = 2 * 15 * W
    src = 2 * H * 8 // 128
    keys = int(2 * H * key_word) // 128
    last = W * (8 * 4 if grouped else sum((1 << u) * min(32, 1 << (u + 1)) for u in range(4)))
    return work + acc + twc + src + keys + last


# FP64 issue cycles of the same CTA-digit: 8 warps x DP_PER_THREAD instructions at 2 warp instructions per clock per SM
FP64_CYCLES_PER_CTA_DIGIT = DP_PER_THREAD * 8 / 2
for n in args.n:
    host = (rng.integers(0, 1 << 62, (n, 3, k, N), dtype=np.uint64) % q[None, None, :, None]).astype(np.uint64)
    a = eng.dev_from(host)
    out = eng.dev_alloc(n * 2 * k * N)
    for _ in range(2):
        eng.raw_relinearize(0, a, n, out)
    eng.sync()
    eng.prof_enable(True)
    eng.timer_start()
    for _ in range(args.iters):
        eng.raw_relinearize(0, a, n, out)
    ms = eng.timer_stop_ms() / args.iters
    prof = eng.prof_collect()
    eng.prof_enable(False)
    fam = {k_: round(v["ms"] / args.iters, 3) for k_, v in prof.items() if v["ms"] > 0}
    fused = prof["ntt_forward"]["launches"] == 0
    w = 8.0 * N
    bytes_digits = w * (n * k * D * 2 + n * k * D + D * 2 * k + n * 2 * k)  # digit source + digits written, digits + keys read, acc written
    key_word = 6.0 if packed else 8.0  # bytes per key word the fused kernel reads (packed copy while every q_l < 2^48)
    bytes_inverse = w * (n * 2 * k * 3)  # acc read, base read, out written (digit path only)
    bytes_fused = w * (n * k + n * 2 * k * 2) + key_word * N * D * 2 * k  # target residues, base read, out written, keys
    cta_digits = n * 2 * k * D
    l2_u64, l2_packed = cta_digits * (8.0 * N + 8.0 * N), cta_digits * (8.0 * N + 6.0 * N)  # source + keys, per key form
    rec = {"n": n, "path": "fused" if fused else "digits", "ms": round(ms, 3), "us_per_ct": round(ms * 1e3 / n, 2), "families_ms": fam,
           "hbm_bytes": {"digits_path": bytes_digits + bytes_inverse, "fused_path": bytes_fused}}
    if fused and fam.get("keyswitch_mac"):
        rate = DP_WARP_INSTR_PER_CT * n / (fam["keyswitch_mac"] * 1e-3)
        rec["fused_fp64_warp_instr_per_s"] = float("%.4g" % rate)
        rec["fused_fp64_issue_share"] = round(rate / 522.7e9, 3)  # 132 SMs x 2 FP64 warp instructions / clock x 1.98 GHz
        # modelled L1 data-path load next to the FP64 pipe's, per CTA-digit: the library reads the grouped last-pass twiddles
        wf = {lay: l1_wavefronts_per_cta_digit(key_word, lay == "grouped") for lay in ("strided", "grouped")}
        rec["model_l1_wavefronts_per_cta_digit"] = wf
        rec["model_l1_cycles_per_fp64_cycle"] = {lay: round(v / FP64_CYCLES_PER_CTA_DIGIT, 3) for lay, v in wf.items()}
        l2 = l2_packed if packed else l2_u64
        rec["fused_l2_bytes"] = {"u64_keys": l2_u64, "packed_keys": l2_packed}
        rec["fused_l2_tb_s"] = round(l2 / (fam["keyswitch_mac"] * 1e-3) / 1e12, 2)
        rec["fused_l2_share"] = round(rec["fused_l2_tb_s"] / args.l2_tbs, 3)
    print(json.dumps(rec), flush=True)
    eng.dev_free(a)
    eng.dev_free(out)
eng.close()
