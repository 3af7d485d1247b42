"""Strided device puts (TensorStore.put of a column slice, read in place by the fused put kernel) against a put of the
slice made contiguous first, on one GPU.

    python bench/strided_put_bench.py [--iters 20] [--warmup 3]

A [16384, 8192] bf16 weight (256 MiB, rows of 16 KiB) is sliced along dim 1 at 1/2, 1/8 and 1/64 of a row (8 KiB, 2 KiB
and 256 B per row), and a [1048576, 128] bf16 tensor (256 B rows) at half a row: 128 B segments, 128 per tile, which is
where the gathering producer issues the most bulk loads per tile.  Each slice is stored into this GPU's HBM slab with XXH3
and with no checksum.  For each (algorithm, shape) it reports the time per call (host clock around a call that ends in a
device synchronise) and the delivered GB/s (object bytes / time) of
  - put(view):        TensorStore.put(W[:, a:b]) -- batch_put_device_strided, the rows gathered by the put kernel,
  - put(contiguous):  TensorStore.put(W[:, a:b].contiguous()) -- a device copy into a temporary, then the plain put.
The key is removed between calls, so every call allocates and writes a fresh object.  After the timed calls a get of
each key is compared with the contiguous slice.  Prints one JSON line per row with the card name and power limit beside
them.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

MiB = 1 << 20


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch

    from blackbird_b200 import _bb
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    if not torch.cuda.is_available():
        sys.exit("strided_put_bench needs a GPU")
    name, power = card()
    cl = GpuRankCluster(slab_bytes=3 * 256 * MiB, cluster_id="strided-put-bench")
    try:
        g = torch.Generator(device="cuda").manual_seed(3)
        tensors = {"weight": torch.randn(16384, 8192, device="cuda", generator=g).to(torch.bfloat16),
                   "kv": torch.randn(1 << 20, 128, device="cuda", generator=g).to(torch.bfloat16)}
        # (tensor, columns [a, b), label)
        shapes = [("weight", 0, 4096, "1/2 row"), ("weight", 1024, 2048, "1/8 row"), ("weight", 4096, 4224, "1/64 row"),
                  ("kv", 0, 64, "1/2 row, 128 segments per tile")]
        rows = []
        for algo in ("XXH3", "NONE"):
            store = TensorStore(cl.client, _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0,
                                                            checksum=getattr(_bb.ChecksumAlgo, algo),
                                                            preferred_classes=[_bb.StorageClass.RAM_GPU]))
            for k, a, b, label in shapes:
                t = tensors[k]
                view = t[:, a:b]
                assert store._gatherable(view) is not None, label
                want = view.contiguous()
                for method, make in (("put(view)", lambda: view), ("put(contiguous)", lambda: view.contiguous())):
                    key = f"{algo}/{k}/{a}/{method}"

                    def call():
                        store.remove([key])
                        store.put(key, make())
                        torch.cuda.synchronize()

                    for _ in range(args.warmup):
                        call()
                    t0 = time.perf_counter()
                    for _ in range(args.iters):
                        call()
                    dt = (time.perf_counter() - t0) / args.iters
                    assert torch.equal(store.get(key), want), (algo, k, a, b, method)
                    n = want.numel() * want.element_size()
                    rows.append({"algo": algo, "tensor": list(t.shape), "columns": [a, b], "shape": label, "row_bytes": (b - a) * 2,
                                 "object_bytes": n, "method": method, "ms_per_call": round(dt * 1e3, 4),
                                 "delivered_GBps": round(n / dt / 1e9, 3)})
                    store.remove([key])
        for r in rows:
            r.update({"gpu": name, "power_limit": power})
            print(json.dumps(r))
    finally:
        cl.stop()


if __name__ == "__main__":
    main()
