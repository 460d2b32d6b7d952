"""Multi-client LoLa serving: images/s and per-batch latency of B clients' inferences run together (networks.serve_batch), each client
with its own secret key and compact key set in a key slot of one server context.

    python tools/lola_batch_bench.py [--nets lola_small,lola,lola_dense,lola_cifar] [--batches 1,8,32,128] [--reps 3]
                                     [--dense-method rows,folded]

Timing: CUDA events on the server context around serve_batch, after one warm-up batch of every B.  Also reported: the share of
key-switch launches that took the fused kernel (cnhe_prof_collect in a separate, untimed pass; INFERRED, not counted: the fused
kernel runs its inverse transforms itself, so the inverse-transform launches (family 1) are taken as digit-path key switches -- at
N = 16384 the multiplies' inverse transforms are counted there too), the device time per kernel family in that profiled pass, and the
card name, power limit and maximum SM clock from nvidia-smi (queries only).  Prints one JSON line per (net, B).  Every network runs with
the reference's parameters (lola_small, LoLa-Dense and LoLa-CIFAR with their SmallModulusCount; timing does not need the scores to
decrypt).  --dense-method: the Method of the score layer of lola_small and LoLa-CIFAR ("rows", the reference's, and / or "folded"), the
methods alternating at every B; score_bytes is the size of the output ciphertexts a batch downloads."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001 -- the figures are still worth printing without the card line
        return dict(gpu="unknown (%s)" % e)


def setup(net_name, B, method="rows"):
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.interfaces import EMatrixFormat
    from cryptonets_b200 import networks as nw
    w60 = dict(DecompositionBitCount=60, GaloisDecompositionBitCount=60)
    if net_name == "lola_small":
        build, primes, n, kw, count, imgs = nw.lola_small, nw.LOLA_SMALL_PRIMES, 8192, dict(DecompositionBitCount=40, GaloisDecompositionBitCount=40), 3, \
            nw.synthetic_mnist(B, seed=1)
    elif net_name == "lola":
        build, primes, n, kw, count, imgs = nw.lola, nw.LOLA_PRIMES, 8192, {}, -1, nw.synthetic_mnist(B, seed=1)
    elif net_name == "lola_dense":
        build, primes, n, kw, count, imgs = nw.lola_dense, nw.LOLA_DENSE_PRIMES, 16384, w60, 7, nw.synthetic_mnist(B, seed=1)
    else:
        build, primes, n, kw, count, imgs = nw.lola_cifar, nw.CIFAR_PRIMES, 16384, dict(DecompositionBitCount=60, GaloisDecompositionBitCount=60), 8, \
            nw.synthetic_cifar(B, seed=1)
    if method != "rows" and net_name not in ("lola_small", "lola_cifar"):
        raise SystemExit("--dense-method applies to lola_small and lola_cifar")
    method_kw = {} if method == "rows" else dict(dense_method=method) if net_name == "lola_small" else dict(score_method=method)
    server, inputs = None, []
    for j in range(B):
        c = B200BfvFactory(primes, n, SmallModulusCount=count, seed=1000 + j, **kw)
        _, rd = build(c, imgs[j:j + 1])
        m = rd.GetNext()
        keys, cts = c.SaveCompactKeys(), c.GetEncryptedMatrixCompact(m.Data, EMatrixFormat.ColumnMajor, 1)
        c.Dispose()
        if server is None:
            server, slot = B200BfvFactory(keys), 0
        else:
            slot = server.AddClientKeys(keys)
        inputs.append((cts, slot, m.Scale))
    net, _ = build(server, imgs[:1], **method_kw)
    return server, net, inputs


def load(server, inputs):
    from cryptonets_b200.interfaces import EMatrixFormat
    ms = []
    for cts, slot, scale in inputs:
        m = server.LoadCompactMatrix(cts, EMatrixFormat.ColumnMajor, slot=slot)
        m.RegisterScale(scale)
        ms.append(m)
    return ms


def run(server, net, inputs):
    from cryptonets_b200.networks import serve_batch
    ms = load(server, inputs)
    eng = server.engine
    eng.timer_start()
    outs = serve_batch(net, ms)
    ms_time = eng.timer_stop_ms()
    score_bytes = sum(v.vec.blocks for m in outs for v in m.vectors) * eng.P * 2 * len(eng.q) * eng.N * 8
    for m in outs + ms:
        m.Dispose()
    return ms_time, score_bytes


def fused_share(server, net, inputs):
    from cryptonets_b200.networks import serve_batch
    ms = load(server, inputs)
    eng = server.engine
    eng.sync()
    eng.prof_enable(True)
    outs = serve_batch(net, ms)
    eng.sync()
    prof = eng.prof_collect()
    eng.prof_enable(False)
    for m in outs + ms:
        m.Dispose()
    ks = prof["keyswitch_mac"]["launches"]
    # per key switch the digit path launches one MAC and one inverse-add; the only other inverse transforms of these networks are the
    # plain multiplies', which do not run under a profiling scope
    digit = min(prof["ntt_inverse"]["launches"], ks)
    return (ks - digit) / ks if ks else 0.0, ks, {k: round(v["ms"], 2) for k, v in prof.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nets", default="lola_small,lola_cifar")
    ap.add_argument("--batches", default="1,8,32,128")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dense-method", default="rows")
    args = ap.parse_args()
    info = card()
    print(json.dumps(info), flush=True)
    for net_name in args.nets.split(","):
        for B in [int(x) for x in args.batches.split(",")]:
            for method in args.dense_method.split(","):
                server, net, inputs = setup(net_name, B, method)
                run(server, net, inputs)  # warm-up of this B
                runs = [run(server, net, inputs) for _ in range(args.reps)]
                times = sorted(r[0] for r in runs)
                share, ks, families = fused_share(server, net, inputs)
                med = times[len(times) // 2]
                print(json.dumps(dict(net=net_name, dense_method=method, B=B, batch_ms=round(med, 2), images_per_s=round(1000.0 * B / med, 1),
                                      keyswitch_launches=ks, score_bytes=runs[0][1], fused_share=round(share, 3), family_ms=families,
                                      reps=args.reps, **info)), flush=True)
                server.Dispose()


if __name__ == "__main__":
    main()
