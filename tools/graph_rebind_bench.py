"""One recorded inference serving four clients (include/cnhe.h cnhe_graph_bind, he.py CapturedInference.Run) against the alternatives, per
network.

    python tools/graph_rebind_bench.py [--nets lola_small_rows,lola_small_folded,lola,lola_cifar,cryptonets_mnist] [--iters 10]
                                       [--rounds 3] [--out results.jsonl]

Setup: a server context holding four clients' compact key sets (key slots), one encrypted input per client, clients served round robin.
Per inference, a host clock around `iters` inferences ending in a device synchronise, the arms alternating in every round, the
median of the rounds (after a warm-up of every arm):
- eager: the layers after the EncryptLayer, Apply by Apply, under the client's slot;
- rebound: one graph recorded for client 0, run for each client in turn (CapturedInference.Run: bind + retag + assign + launch; the
  synchronise ends the window, so a run's host work overlaps the previous launch);
- control: the same graph run for client 0 only (Run binds it to the slot it already has: no retag, no table copy);
- rebound_sync / control_sync: the same two, each inference followed by a device synchronise (the latency of one request on its own).
It also reports what one recording per client would cost: the wall time of one CaptureInference and its device bytes, against one
graph's bytes; whether every rebound replay's words equal the eager words; and the card's name, power limit and maximum SM clock, from
nvidia-smi in the same run.  Prints one JSON line per network (and appends it to --out)."""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.graph_replay_bench import card  # noqa: E402

CLIENTS = 4


def setup(name):
    """(factory, net): the server factory and the network"""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200 import networks as nw
    if name.startswith("lola_small"):
        f = B200BfvFactory(nw.LOLA_SMALL_PRIMES, 8192, DecompositionBitCount=40, GaloisDecompositionBitCount=40, SmallModulusCount=3, seed=5)
        return f, nw.lola_small(f, nw.synthetic_mnist(2, seed=6), dense_method=name.split("_")[-1])
    if name == "lola":
        f = B200BfvFactory(nw.LOLA_PRIMES, 8192, seed=5)
        return f, nw.lola(f, nw.synthetic_mnist(2, seed=6))
    if name == "lola_cifar":
        f = B200BfvFactory(nw.CIFAR_PRIMES, 16384, DecompositionBitCount=60, GaloisDecompositionBitCount=60, SmallModulusCount=8, seed=5)
        return f, nw.lola_cifar(f, nw.synthetic_cifar(2), dense_method="diagonal", score_method="folded")
    if name == "cryptonets_mnist":
        f = B200BfvFactory(nw.CRYPTONETS_PRIMES, 8192, seed=77)
        return f, nw.cryptonets_mnist(f, nw.synthetic_mnist(8192, seed=8), batch_size=8192)
    raise SystemExit("unknown network " + name)


def run(name, iters, rounds):
    from cryptonets_b200.he import B200BfvMatrix
    from cryptonets_b200.layers import EncryptLayer, TimingLayer
    f, (net, rd) = setup(name)
    eng = f.engine
    net.PrepareNetwork()
    chain, layer = [], net
    while not isinstance(layer, EncryptLayer):
        if not isinstance(layer, TimingLayer):
            chain.append(layer)
        layer = layer.Source
    chain.reverse()
    x = layer.Apply(rd.GetNext())
    galois = [] if name == "cryptonets_mnist" else None
    slots = [f.AddClientKeys(f.SaveCompactKeys(public=False, galois=galois)) for _ in range(CLIENTS)]

    def in_slot(s):
        m = B200BfvMatrix(f, x.vectors, x.Format)
        for v in m.vectors:
            v.vec.set_key_slot(s)
        return m

    ins = [in_slot(s) for s in slots]

    def eager(m):
        cur = m
        for lay in chain:
            out = lay.Apply(cur)
            if out is not cur and cur is not m:
                cur.Dispose()
            cur = out
        return cur

    want = []
    for m in ins:
        out = eager(m)
        want.append(eng.export_raw_many([v.vec for v in out.vectors]))
        out.Dispose()
    # the alternative: one recording per client (each recorded, measured and released in turn)
    capture_ms, per_client_bytes = [], []
    for s in slots:
        eng.sync()
        t0 = time.perf_counter()
        c = f.CaptureInference(net, in_slot(s))
        eng.sync()
        capture_ms.append((time.perf_counter() - t0) * 1e3)
        per_client_bytes.append(c.Info()["device_bytes"])
        c.Dispose()
    cap = f.CaptureInference(net, in_slot(slots[0]))
    same = True
    for j, m in enumerate(ins):
        out = cap.Run(m)
        same = same and bool((eng.export_raw_many([v.vec for v in out.vectors]) == want[j]).all())

    def eager_arm(j):
        eager(ins[j % CLIENTS]).Dispose()

    def rebound_arm(j):
        cap.Run(ins[j % CLIENTS])

    def control_arm(j):
        cap.Run(ins[0])

    def rebound_sync_arm(j):
        cap.Run(ins[j % CLIENTS])
        eng.sync()

    def control_sync_arm(j):
        cap.Run(ins[0])
        eng.sync()

    arms = dict(eager=eager_arm, rebound=rebound_arm, control=control_arm, rebound_sync=rebound_sync_arm, control_sync=control_sync_arm)
    for fn in arms.values():  # warm-up
        for j in range(CLIENTS):
            fn(j)
    eng.sync()
    times = {a: [] for a in arms}
    for _ in range(rounds):
        for a, fn in arms.items():
            eng.sync()
            t0 = time.perf_counter()
            for j in range(iters):
                fn(j)
            eng.sync()
            times[a].append((time.perf_counter() - t0) * 1e3 / iters)
    info = cap.Info()
    cap.Dispose()
    f.Dispose()
    res = dict(network=name, clients=CLIENTS, iters=iters, rounds=rounds, words_equal_eager=same, graph_device_bytes=info["device_bytes"],
               per_client_capture_ms=[round(t, 1) for t in capture_ms], per_client_device_bytes=per_client_bytes)
    for a in arms:
        res[a + "_ms"] = round(statistics.median(times[a]), 3)
        res[a + "_ms_rounds"] = [round(t, 3) for t in times[a]]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nets", default="lola_small_rows,lola_small_folded,lola,lola_cifar,cryptonets_mnist")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    c = card()
    for name in a.nets.split(","):
        res = dict(run(name, a.iters, a.rounds), **c)
        line = json.dumps(res)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as fh:
                fh.write(line + "\n")


if __name__ == "__main__":
    main()
