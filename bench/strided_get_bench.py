"""Strided device gets (TensorStore.get_slice along dim 1) against a whole get followed by narrow().contiguous(), on one GPU.

    python bench/strided_get_bench.py [--iters 20] [--warmup 3]

A [16384, 8192] bf16 weight (256 MiB, rows of 16 KiB) stored whole in this GPU's HBM slab, written with XXH3 and with no
checksum, sliced along dim 1 at 1/2, 1/8 and 1/64 of a row (8 KiB, 2 KiB and 256 B per row).  The kernel stores one row
segment per lane; with a 16 KiB pitch a tile holds at most two segments, so a [1048576, 128] bf16 tensor (256 B rows,
64 segments per tile) sliced at half a row is measured too.  Columns [0, 4093) of the weight leave a 6-byte gap between
rows, which the fused kernel cannot store co-aligned: that shape is staged through the host.  For each (algorithm,
shape) it reports the time per call (host clock around a call that ends in a device synchronise) and the delivered GB/s
(result bytes / time) of
  - get_slice:     TensorStore.get_slice (the strided device get: one read of the object, rows * width bytes written),
  - whole+narrow:  TensorStore.get of the whole tensor, then .narrow(1, a, b - a).contiguous() (a full temporary written
                   and read back).
A verified strided read reads the whole object; without a checksum only the aligned span from the first row to the last.
Prints one JSON line per row with the card name and power limit beside them.
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
    ap.add_argument("--staged-iters", type=int, default=3)
    args = ap.parse_args()

    import torch

    from blackbird_b200 import _bb
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    if not torch.cuda.is_available():
        sys.exit("strided_get_bench needs a GPU")
    name, power = card()
    cl = GpuRankCluster(slab_bytes=5 * 256 * MiB, cluster_id="strided-bench")
    try:
        g = torch.Generator(device="cuda").manual_seed(3)
        tensors = {"weight": torch.randn(16384, 8192, device="cuda", generator=g).to(torch.bfloat16),
                   "kv": torch.randn(1 << 20, 128, device="cuda", generator=g).to(torch.bfloat16)}
        # (tensor, columns [a, b), label)
        shapes = [("weight", 0, 4096, "1/2 row"), ("weight", 1024, 2048, "1/8 row"), ("weight", 4096, 4224, "1/64 row"),
                  ("kv", 0, 64, "1/2 row, 64 rows per tile"), ("weight", 0, 4093, "6-byte gap: host-staged")]
        rows = []
        for algo in ("XXH3", "NONE"):
            store = TensorStore(cl.client, _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0,
                                                            checksum=getattr(_bb.ChecksumAlgo, algo),
                                                            preferred_classes=[_bb.StorageClass.RAM_GPU]))
            for k, t in tensors.items():
                store.put(f"{algo}/{k}", t)
            for k, a, b, label in shapes:
                key, t = f"{algo}/{k}", tensors[k]
                want = t[:, a:b].contiguous()
                out = {}

                def sliced():
                    out["t"] = store.get_slice(key, 1, a, b)
                    torch.cuda.synchronize()

                def whole_narrow():
                    out["t"] = store.get(key).narrow(1, a, b - a).contiguous()
                    torch.cuda.synchronize()

                staged = "staged" in label
                for method, fn in (("get_slice", sliced), ("whole+narrow", whole_narrow)):
                    iters = min(args.iters, args.staged_iters) if staged and method == "get_slice" else args.iters
                    for _ in range(args.warmup):
                        fn()
                    t0 = time.perf_counter()
                    for _ in range(iters):
                        fn()
                    dt = (time.perf_counter() - t0) / iters
                    assert torch.equal(out["t"], want), (algo, k, a, b, method)
                    n = want.numel() * want.element_size()
                    rows.append({"algo": algo, "tensor": list(t.shape), "columns": [a, b], "shape": label, "row_bytes": (b - a) * 2,
                                 "result_bytes": n, "method": method, "ms_per_call": round(dt * 1e3, 4),
                                 "delivered_GBps": round(n / dt / 1e9, 3)})
        for r in rows:
            r.update({"gpu": name, "power_limit": power})
            print(json.dumps(r))
    finally:
        cl.stop()


if __name__ == "__main__":
    main()
