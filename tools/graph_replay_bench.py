"""Latency of one inference, eager layer calls against one replay of the recorded graph (he.py CaptureInference, include/cnhe.h
cnhe_capture_begin), per network.

    python tools/graph_replay_bench.py [--nets lola_small_rows,lola_small_folded,lola_small_b8,lola,lola_cifar,cryptonets_mnist]
                                       [--iters 20] [--rounds 3] [--out results.jsonl]

Per network:
- wall time per inference: a host clock around `iters` inferences ending in a device synchronise, eager and replay alternating in every
  round, the median of the rounds (after a warm-up of both arms).  The eager arm is the layers after the EncryptLayer, Apply by Apply
  (serve_batch's ApplyBatch for lola_small_b8, eight clients in key slots); the replay arm assigns the input and launches the graph.
- device-busy time per inference: the union of the kernel, memcpy and memset intervals in a torch.profiler (CUDA activities) trace of
  one profiled pass of each arm, run separately from the timed rounds, divided by the inferences in the pass.
- kernels per inference (cnhe_kernel_launch_count of the eager arm; the graph's kernel nodes), the graph's device bytes, and whether the
  replay's output words equal the eager ones.
- the card's name, power limit and maximum SM clock, from nvidia-smi queries in the same run.
Prints one JSON line per network (and appends it to --out)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001 -- the figures are still worth printing without the card line
        return dict(gpu="unknown (%s)" % e)


def _chain(net):
    from cryptonets_b200.layers import EncryptLayer, TimingLayer
    chain, layer = [], net
    while not isinstance(layer, EncryptLayer):
        if not isinstance(layer, TimingLayer):
            chain.append(layer)
        layer = layer.Source
    return layer, chain[::-1]


def setup(name):
    """(factory, net, input A, input B, batch): inputs are one encrypted matrix, or a list of eight (one per client) for lola_small_b8"""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.interfaces import EMatrixFormat
    from cryptonets_b200 import networks as nw
    w40 = dict(DecompositionBitCount=40, GaloisDecompositionBitCount=40, SmallModulusCount=3)
    if name == "lola_small_b8":
        imgs = nw.synthetic_mnist(16, seed=1)
        f = B200BfvFactory(nw.LOLA_SMALL_PRIMES, 8192, seed=999, **w40)
        sets = [[], []]
        for j in range(8):
            c = B200BfvFactory(nw.LOLA_SMALL_PRIMES, 8192, seed=1000 + j, **w40)
            _, rd = nw.lola_small(c, imgs)
            slot = f.AddClientKeys(c.SaveCompactKeys(public=False))
            for r in range(2):
                rd.pos = j + 8 * r
                m = rd.GetNext()
                x = f.LoadCompactMatrix(c.GetEncryptedMatrixCompact(m.Data, EMatrixFormat.ColumnMajor, 1), EMatrixFormat.ColumnMajor, slot=slot)
                x.RegisterScale(m.Scale)
                sets[r].append(x)
            c.Dispose()
        net, _ = nw.lola_small(f, imgs[:1])
        net.PrepareNetwork()
        return f, net, sets[0], sets[1], True
    if name.startswith("lola_small"):
        f = B200BfvFactory(nw.LOLA_SMALL_PRIMES, 8192, seed=5, **w40)
        net, rd = nw.lola_small(f, nw.synthetic_mnist(2, seed=6), dense_method=name.split("_")[-1])
    elif name == "lola":
        f = B200BfvFactory(nw.LOLA_PRIMES, 8192, seed=5)
        net, rd = nw.lola(f, nw.synthetic_mnist(2, seed=6))
    elif name == "lola_cifar":
        f = B200BfvFactory(nw.CIFAR_PRIMES, 16384, DecompositionBitCount=60, GaloisDecompositionBitCount=60, SmallModulusCount=8, seed=5)
        net, rd = nw.lola_cifar(f, nw.synthetic_cifar(2), dense_method="diagonal", score_method="folded")
    elif name == "cryptonets_mnist":
        f = B200BfvFactory(nw.CRYPTONETS_PRIMES, 8192, seed=77)
        net, rd = nw.cryptonets_mnist(f, nw.synthetic_mnist(2 * 8192, seed=8), batch_size=8192)
    else:
        raise SystemExit("unknown network " + name)
    net.PrepareNetwork()
    enc, _ = _chain(net)
    return f, net, enc.Apply(rd.GetNext()), enc.Apply(rd.GetNext()), False


def eager(net, x, batch):
    from cryptonets_b200.networks import serve_batch
    if batch:
        return serve_batch(net, x)
    cur = x
    for layer in _chain(net)[1]:
        out = layer.Apply(cur)
        if out is not cur and cur is not x:
            cur.Dispose()
        cur = out
    return cur


def words(f, out, batch):
    import numpy as np
    return np.concatenate([f.engine.export_raw_many([v.vec for v in m.vectors]).ravel() for m in (out if batch else [out])])


def dispose(out, batch):
    for m in (out if batch else [out]):
        m.Dispose()


def busy_ms(fn, iters):
    """device-busy milliseconds per call of fn: the union of the device activity intervals of a profiled pass"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                fn()
            torch.cuda.synchronize()
        prof.export_chrome_trace(path)
        ev = json.load(open(path))
        ev = ev["traceEvents"] if isinstance(ev, dict) else ev
    spans = sorted((e["ts"], e["ts"] + e.get("dur", 0)) for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset"))
    total, end = 0.0, None
    for a, b in spans:
        if end is None or a > end:
            total += b - a
            end = b
        elif b > end:
            total += b - end
            end = b
    return total / 1000.0 / iters, len(spans) / iters


def bench(name, iters, rounds):
    f, net, xa, xb, batch = setup(name)
    eng = f.engine
    try:
        want = eager(net, xb, batch)
        ref = words(f, want, batch)
        dispose(want, batch)
        k0 = eng.launch_count()
        dispose(eager(net, xa, batch), batch)
        eng.sync()
        kernels = eng.launch_count() - k0
        cap = f.CaptureInference(net, xa)
        info = cap.Info()
        same = bool((words(f, cap.Run(xb), batch) == ref).all())

        def run_eager():
            dispose(eager(net, xb, batch), batch)

        def run_replay():
            cap.Run(xb)

        def timed(fn):
            eng.sync()
            t0 = time.perf_counter()
            for _ in range(iters):
                fn()
            eng.sync()
            return (time.perf_counter() - t0) * 1000.0 / iters

        timed(run_eager), timed(run_replay)  # warm-up
        e_ms, r_ms = [], []
        for _ in range(rounds):
            e_ms.append(timed(run_eager))
            r_ms.append(timed(run_replay))
        e_busy, e_act = busy_ms(run_eager, max(1, iters // 4))
        r_busy, r_act = busy_ms(run_replay, max(1, iters // 4))
        e_wall, r_wall = statistics.median(e_ms), statistics.median(r_ms)
        cap.Dispose()
        return dict(net=name, iters=iters, rounds=rounds, eager_ms=round(e_wall, 3), replay_ms=round(r_wall, 3), eager_rounds_ms=[round(x, 3) for x in e_ms],
                    replay_rounds_ms=[round(x, 3) for x in r_ms], speedup=round(e_wall / r_wall, 3),
                    eager_busy_ms=round(e_busy, 3), replay_busy_ms=round(r_busy, 3), eager_busy_share=round(e_busy / e_wall, 3),
                    replay_busy_share=round(r_busy / r_wall, 3), eager_device_activities=round(e_act, 1), replay_device_activities=round(r_act, 1),
                    kernels_per_inference=kernels, graph_kernel_nodes=info["kernel_nodes"], graph_device_bytes=info["device_bytes"],
                    replay_words_equal_eager=same, **card())
    finally:
        f.Dispose()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nets", default="lola_small_rows,lola_small_folded,lola_small_b8,lola,lola_cifar,cryptonets_mnist")
    ap.add_argument("--iters", type=int, default=20, help="inferences per timed round (CryptoNets' 8192-image batch: a quarter)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    for name in a.nets.split(","):
        r = bench(name, max(2, a.iters // 4) if name == "cryptonets_mnist" else a.iters, a.rounds)
        line = json.dumps(r)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as fh:
                fh.write(line + "\n")


if __name__ == "__main__":
    main()
