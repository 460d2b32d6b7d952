"""Levelled replays on an H100: one inference per arm -- eager unlevelled, eager levelled, replay unlevelled, replay levelled (he.py
CaptureInference, SpanLevels=True for the levelled graph; include/cnhe.h cnhe_capture_begin_levels) -- per network.

    python tools/graph_levels_bench.py [--nets lola,lola_dense,lola_cifar] [--iters 10] [--rounds 3] [--out results.jsonl]

Per network, at level_bench's test parameters with the committed schedule (networks.LEVEL_SCHEDULES):
- wall time per inference: a host clock around `iters` inferences ending in a synchronise of every context of the family, the four arms
  alternating in every round, the median of the rounds (after a warm-up of every arm);
- device-busy time per inference: graph_replay_bench.busy_ms, one profiled pass per arm, run separately from the timed rounds;
- the graphs' kernel nodes and device bytes, the eager arms' kernel launches, and whether each replay's words equal its eager arm's;
- lola only: four compact-key clients served round robin by the levelled graph, each request rebound (one client added to the server after
  the recording, so its first bind restricts its keys into the levels), against the same requests served eagerly;
- the card's name, power limit and maximum SM clock, read in the same run.
LoLa-CIFAR runs with dense_method="diagonal", score_method="folded"; when the device runs out of memory it is reported as not measured.
Prints one JSON line per network (and appends it to --out)."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import graph_replay_bench as GR  # noqa: E402
import level_bench as LB  # noqa: E402
from cryptonets_b200._lib import CnheError  # noqa: E402
from cryptonets_b200.networks import LEVEL_SCHEDULES  # noqa: E402

KWARGS = {"lola_cifar": dict(dense_method="diagonal", score_method="folded")}


def _eager(chain, x):
    return LB.run(chain, x)


def _words(m):
    return m.factory.engine.export_raw_many([v.vec for v in m.vectors])


def _in_slot(f, m, slot):
    from cryptonets_b200.he import B200BfvMatrix
    c = B200BfvMatrix(f, m.vectors, m.Format)
    for v in c.vectors:
        v.vec.set_key_slot(slot)
    return c


def bench(name, iters, rounds):
    build = LB.NETS[name][0]
    f = LB.factory(name)
    try:
        imgs = (LB.nw.synthetic_cifar if name == "lola_cifar" else LB.nw.synthetic_mnist)(2, seed=6)
        kw = KWARGS.get(name, {})
        nets = {"full": build(f, imgs, **kw)[0], "levels": build(f, imgs, levels=LEVEL_SCHEDULES[name], **kw)[0]}
        chains = {k: LB.chain_of(n) for k, n in nets.items()}
        xa, xb = LB.encrypted_input(f, name, imgs[:1]), LB.encrypted_input(f, name, imgs[1:2])  # set-up input, timed input
        res = dict(net=name, schedule=LEVEL_SCHEDULES[name], iters=iters, rounds=rounds)
        kernels, want = {}, {}
        for k, c in chains.items():
            _eager(c, xa).Dispose()  # set-up: levels, plans
            LB.sync(f)
            k0 = sum(g.engine.launch_count() for g in LB.family(f))
            out = _eager(c, xb)
            want[k] = _words(out)
            out.Dispose()
            kernels[k] = sum(g.engine.launch_count() for g in LB.family(f)) - k0
        caps = {k: f.CaptureInference(n, LB.encrypted_input(f, name, imgs[:1]), SpanLevels=(k == "levels")) for k, n in nets.items()}
        res["kernels_per_inference"] = kernels
        res["graph"] = {k: c.Info() for k, c in caps.items()}
        res["replay_words_equal_eager"] = {k: bool((_words(caps[k].Run(xb)) == want[k]).all()) for k in caps}
        arms = {"eager_full": lambda: _eager(chains["full"], xb).Dispose(), "eager_levels": lambda: _eager(chains["levels"], xb).Dispose(),
                "replay_full": lambda: caps["full"].Run(xb), "replay_levels": lambda: caps["levels"].Run(xb)}

        def timed(fn):
            LB.sync(f)
            t0 = time.perf_counter()
            for _ in range(iters):
                fn()
            LB.sync(f)
            return (time.perf_counter() - t0) * 1000.0 / iters

        for fn in arms.values():
            timed(fn)
        ms = {k: [] for k in arms}
        for _ in range(rounds):
            for k, fn in arms.items():
                ms[k].append(timed(fn))
        res["ms_per_inference"] = {k: round(statistics.median(v), 3) for k, v in ms.items()}
        res["ms_rounds"] = {k: [round(x, 3) for x in v] for k, v in ms.items()}
        res["busy_ms_per_inference"] = {k: round(GR.busy_ms(fn, max(2, iters // 2))[0], 3) for k, fn in arms.items()}
        if name == "lola":
            res["rebind"] = rebind(f, chains["levels"], caps["levels"], imgs, iters)
        for c in caps.values():
            c.Dispose()
        return res
    finally:
        f.Dispose()


def rebind(f, chain, cap, imgs, iters):
    """four compact-key clients, added to the server after the recording, round robin through the levelled graph with each request rebound,
    and the same requests eagerly; ms per request with a synchronise of the family after each.  Three clients reach the levels through an
    eager run first; the fourth only through the graph's bind, whose first run is timed on its own."""
    slots = [f.AddClientKeys(f.SaveCompactKeys(public=False)) for _ in range(4)]
    x = LB.encrypted_input(f, "lola", imgs[:1])
    ins = [_in_slot(f, x, s) for s in slots]
    for m in ins[:3]:  # the first three clients reach the levels through an eager switch; the fourth only through the graph's bind
        _eager(chain, m).Dispose()
    first = time.perf_counter()
    got = _words(cap.Run(ins[3]))
    first_ms = (time.perf_counter() - first) * 1000.0
    out = _eager(chain, ins[3])
    same = bool((got == _words(out)).all())
    out.Dispose()

    def serve(fn):
        LB.sync(f)
        t0 = time.perf_counter()
        for i in range(iters):
            fn(ins[i % 4])
            LB.sync(f)
        return (time.perf_counter() - t0) * 1000.0 / iters

    replay = lambda m: cap.Run(m)
    eager = lambda m: _eager(chain, m).Dispose()
    serve(replay), serve(eager)
    r, e = [], []
    for _ in range(3):
        r.append(serve(replay))
        e.append(serve(eager))
    return dict(clients=4, late_client_first_run_ms=round(first_ms, 3), late_client_words_equal_eager=same,
                replay_rebound_ms=round(statistics.median(r), 3), eager_ms=round(statistics.median(e), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nets", default="lola,lola_dense,lola_cifar")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    card = GR.card()
    for name in a.nets.split(","):
        try:
            r = bench(name, a.iters, a.rounds)
        except CnheError as e:
            if "memory" not in str(e).lower():
                raise
            r = dict(net=name, note="not measured: out of device memory (%s)" % e)
        r.update(card)
        line = json.dumps(r)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as fh:
                fh.write(line + "\n")


if __name__ == "__main__":
    main()
