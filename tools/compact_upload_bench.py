"""CryptoNets-MNIST end-to-end serving loop with raw and with compact ciphertext uploads, alternated in one process.

The loop is bench.py's e2e leg: pinned host buffers, multi-stream, pipeline depth 1 (batch i+1 is imported before the scores of batch i
are waited for).  Raw imports upload 2kN words per ciphertext (cnhe_vecs_import_raw); compact imports upload the bit-packed c0 plus the
per-channel ChaCha20 keys and expand c1 on the GPU (cnhe_vecs_import_compact).  Prints one JSON line:
  e2e images/s and H2D bytes per batch for both, the expansion's device time per batch (CUDA events around k_compact_expand) and its
  bytes/s against HBM (packed bytes read + ciphertext bytes written), the client-side encrypt_compact time per batch, and the card.

  python tools/compact_upload_bench.py [--steps 10] [--repeats 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BATCH = 8192


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # the numbers below are still device-event timed; the card is then unknown
        return dict(error=str(e))


def build_network(factory):
    from cryptonets_b200.layers import PoolLayer, SquareActivation
    from cryptonets_b200.networks import cryptonets_weights, transpose

    class Src:
        Factory = factory

        def GetOutputScale(self):
            return 16.0

        def PrepareNetwork(self):
            pass

    w = cryptonets_weights()
    conv1 = PoolLayer(Source=Src(), InputShape=[28, 28], KernelShape=[5, 5], Upperpadding=[1, 1], Stride=[2, 2], MapCount=[5, 1], WeightsScale=32,
                      Weights=w["Weights_0"])
    act2 = SquareActivation(Source=conv1)
    dense3 = PoolLayer(Source=act2, InputShape=[845], KernelShape=[845], Stride=[1000], MapCount=[100], Weights=transpose(w["Weights_1"], 845, 100),
                       Bias=w["Biases_2"], WeightsScale=1024)
    act4 = SquareActivation(Source=dense3)
    dense5 = PoolLayer(Source=act4, InputShape=[100], KernelShape=[100], Stride=[1000], MapCount=[10], Weights=w["Weights_3"], Bias=w["Biases_3"],
                       WeightsScale=32)
    layers = [conv1, act2, dense3, act4, dense5]
    dense5.PrepareNetwork()
    return layers


def forward(layers, m):
    for layer in layers:
        nxt = layer.Apply(m)
        if layer is not layers[0]:
            m.Dispose()
        m = nxt
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    from cryptonets_b200.he import B200BfvFactory, B200BfvMatrix, B200BfvVector
    from cryptonets_b200.interfaces import EMatrixFormat
    from cryptonets_b200.networks import CRYPTONETS_PRIMES, synthetic_mnist

    f = B200BfvFactory(CRYPTONETS_PRIMES, BATCH, seed=1)
    eng = f.engine
    layers = build_network(f)
    x = np.rint(synthetic_mnist(BATCH, seed=20240917) / 256.0 * 16.0)

    # client side: the compact blob of one batch (timed: encode, seeded encryption, packing, device-to-host)
    f.GetEncryptedMatrixCompact(x, EMatrixFormat.ColumnMajor, 1)
    enc_ms = []
    for _ in range(3):
        eng.sync()
        t0 = time.perf_counter()
        blob = f.GetEncryptedMatrixCompact(x, EMatrixFormat.ColumnMajor, 1)
        enc_ms.append((time.perf_counter() - t0) * 1e3)
    host_c = torch.empty(len(blob), dtype=torch.uint8).pin_memory()
    host_c.numpy()[:] = np.frombuffer(blob, dtype=np.uint8)
    # raw form of the same ciphertexts
    xm = f.LoadCompactMatrix(blob, EMatrixFormat.ColumnMajor)
    host_r = torch.empty(eng.P * 784 * eng.ct_words, dtype=torch.int64).pin_memory()
    eng.export_raw_many([v.vec for v in xm.vectors], host_r.data_ptr())
    xm.Dispose()
    host_out = [torch.empty(eng.P * 10 * eng.ct_words, dtype=torch.int64).pin_memory() for _ in range(2)]
    raw_bytes, compact_bytes = host_r.numel() * 8, len(blob)

    def imp(kind):
        if kind == "raw":
            vecs = eng.import_raw_many(host_r.data_ptr(), 784, 1, BATCH, 16.0)
        else:
            vecs = eng.import_compact(host_c.data_ptr(), compact_bytes)
            for v in vecs:
                v.register_scale(16.0)
        return B200BfvMatrix(f, [B200BfvVector(f, v) for v in vecs], EMatrixFormat.ColumnMajor, CopyVectors=False)

    def e2e_run(kind, steps, depth=1):
        nxt = imp(kind)
        pending = []
        for s_ in range(steps):
            cur = nxt
            out = forward(layers, cur)
            cur.Dispose()
            ticket = eng.export_raw_many_async([v.vec for v in out.vectors], host_out[s_ % (depth + 1)].data_ptr())
            out.Dispose()
            if s_ + 1 < steps:
                nxt = imp(kind)
            pending.append(ticket)
            if len(pending) > depth:
                eng.export_wait(pending.pop(0))
        for t in pending:
            eng.export_wait(t)

    eng.set_option("multi_stream", 1)
    for kind in ("raw", "compact"):
        e2e_run(kind, args.warmup)
    eng.sync()
    rates = {"raw": [], "compact": []}
    for _ in range(args.repeats):
        for kind in ("raw", "compact"):
            eng.sync()
            t0 = time.perf_counter()
            e2e_run(kind, args.steps)
            eng.sync()
            rates[kind].append(BATCH * args.steps / (time.perf_counter() - t0))

    # the expansion alone: device time of k_compact_expand per batch (profiling family "other" holds only it here)
    eng.sync()
    eng.prof_enable(True)
    eng.prof_collect()
    reps = 10
    for _ in range(reps):
        m = imp("compact")
        eng.sync()
        m.Dispose()
    prof = eng.prof_collect()["other"]
    eng.prof_enable(False)
    exp_ms = prof["ms"] / reps
    exp_bytes = prof["bytes"] / reps

    res = dict(
        workload="cryptonets_mnist_e2e_upload", batch=BATCH, steps=args.steps, repeats=args.repeats, card=card(),
        raw=dict(images_per_s=rates["raw"], median=float(np.median(rates["raw"])), h2d_bytes_per_batch=raw_bytes),
        compact=dict(images_per_s=rates["compact"], median=float(np.median(rates["compact"])), h2d_bytes_per_batch=compact_bytes),
        byte_ratio=raw_bytes / compact_bytes,
        expand=dict(ms_per_batch=exp_ms, launches=prof["launches"], hbm_bytes_per_batch=exp_bytes,
                    hbm_gb_per_s=exp_bytes / (exp_ms * 1e-3) / 1e9 if exp_ms > 0 else 0.0),
        client_encrypt_compact_ms_per_batch=enc_ms,
    )
    print(json.dumps(res))
    f.Dispose()


if __name__ == "__main__":
    main()
