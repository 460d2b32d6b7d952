"""Size and speed of compact evaluation-key upload (cnhe_keys_save_compact / cnhe_context_load_compact) for the served parameter sets.

Per set (CryptoNets-MNIST, LoLa-small, LoLa-CIFAR; secure-mode keys) it reports:
  bytes of the reference key archive (cnhe_keys_save without secret keys), of the compact blob with every key and with the selection
  the network needs (CryptoNets never rotates: pk + relinearisation keys; the LoLa networks: every element);
  client export time of the full blob (host clock; the call ends in a synchronise);
  server load time (host clock around cnhe_context_load_compact, which ends in a synchronise; includes creating the context);
  expansion device time: the k_compact_expand kernels of one load, from torch.profiler's CUDA activity;
and the card's name, power limit and max SM clock read in the same run.  Prints one JSON line.

  python tools/compact_keys_bench.py [--repeats 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SETS = {
    "cryptonets_mnist": dict(t=[549764251649, 549764284417], N=8192, count=-1, dbc=(10, 20), needed=[]),
    "lola_small": dict(t=[2277377, 2424833], N=8192, count=3, dbc=(40, 40), needed=None),
    "lola_cifar": dict(t=[957181001729, 957181034497], N=16384, count=8, dbc=(60, 60), needed=None),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # the device times below are still measured; the card is then unknown
        return dict(error=str(e))


def expansion_ms(blob):
    """device time of the k_compact_expand kernels of one cnhe_context_load_compact"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from cryptonets_b200.engine import Engine
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        Engine(None, compact_keys=blob).close()
        torch.cuda.synchronize()
    total, n = 0.0, 0
    for ev in prof.events():
        if "k_compact_expand" in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA:
            total += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            n += 1
    return total / 1000.0, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    from cryptonets_b200.engine import Engine
    res = dict(card=card(), sets={})
    for name, s in SETS.items():
        client = Engine(s["t"], s["N"], s["dbc"][0], s["dbc"][1], s["count"])
        client.keygen(None)
        archive = len(client.save_keys(False))
        exports, blob = [], None
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            blob = client.save_compact_keys()
            exports.append(time.perf_counter() - t0)
        needed = client.save_compact_keys(galois=s["needed"])
        client.close()
        Engine(None, compact_keys=blob).close()  # first load pays for module loading and the memory pool
        loads = []
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            Engine(None, compact_keys=blob).close()
            loads.append(time.perf_counter() - t0)
        dev_ms, kernels = expansion_ms(blob)
        res["sets"][name] = dict(N=s["N"], archive_bytes=archive, compact_every_bytes=len(blob), compact_needed_bytes=len(needed),
                                 ratio_every=round(archive / len(blob), 3), export_s_median=round(sorted(exports)[len(exports) // 2], 4),
                                 load_s_median=round(sorted(loads)[len(loads) // 2], 4), load_s_min=round(min(loads), 4),
                                 expand_device_ms=round(dev_ms, 3), expand_kernels=kernels)
        print(name, res["sets"][name], file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
