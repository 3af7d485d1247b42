"""Gets into a sliced tensor (TensorStore.get_into of a column slice, stored by the scattering store of the fused get
kernel) against what a user writes without it, a get into a fresh tensor and a copy into the slice, on one GPU.

    python bench/scatter_get_bench.py [--iters 20] [--warmup 3]

A [16384, 8192] bf16 weight (256 MiB, rows of 16 KiB) is sliced along dim 1 at 1/2, 1/8 and 1/64 of a row (8 KiB, 2 KiB
and 256 B per row), and a [1048576, 128] bf16 tensor (256 B rows) at half a row: 128 B segments, 128 per tile, which is
where the scattering store warp issues the most bulk stores per tile.  Each slice is stored whole in this GPU's HBM slab
with XXH3, with no checksum, and packed as MXFP8.  For each (storage, shape) it reports the time per call (host clock
around a call that ends in a device synchronise) and the delivered GB/s (bf16 bytes of the slice / time) of
  - get_into(view):  TensorStore.get_into(key, W[:, a:b]) -- batch_get_device_scatter (or the fp8 form), the rows
                     stored by the get kernel,
  - get + copy_:     W[:, a:b].copy_(TensorStore.get(key)) -- a get into a temporary, then a device copy.
After the timed calls the slice is compared with the stored tensor.  Prints one JSON line per row with the card name and
power limit beside them.
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
        sys.exit("scatter_get_bench needs a GPU")
    name, power = card()
    cl = GpuRankCluster(slab_bytes=3 * 256 * MiB, cluster_id="scatter-get-bench")
    try:
        g = torch.Generator(device="cuda").manual_seed(3)
        tensors = {"weight": torch.randn(16384, 8192, device="cuda", generator=g).to(torch.bfloat16),
                   "kv": torch.randn(1 << 20, 128, device="cuda", generator=g).to(torch.bfloat16)}
        # (tensor, columns [a, b), label)
        shapes = [("weight", 0, 4096, "1/2 row"), ("weight", 1024, 2048, "1/8 row"), ("weight", 4096, 4224, "1/64 row"),
                  ("kv", 0, 64, "1/2 row, 128 segments per tile")]
        rows = []
        for storage in ("XXH3", "NONE", "MXFP8"):
            algo = "BBH64" if storage == "MXFP8" else storage
            store = TensorStore(cl.client, _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0,
                                                            checksum=getattr(_bb.ChecksumAlgo, algo),
                                                            preferred_classes=[_bb.StorageClass.RAM_GPU]))
            for k, a, b, label in shapes:
                t = tensors[k]
                key = f"{storage}/{k}/{a}"
                store.put(key, t[:, a:b].contiguous(), pack_fp8=storage == "MXFP8")
                want = store.get(key)
                target = torch.zeros_like(t)
                view = target[:, a:b]
                assert store._source_rows(view) is not None, label

                def into():
                    store.get_into(key, view)
                    torch.cuda.synchronize()

                def get_copy():
                    view.copy_(store.get(key))
                    torch.cuda.synchronize()

                for method, call in (("get_into(view)", into), ("get + copy_", get_copy)):
                    target.zero_()
                    for _ in range(args.warmup):
                        call()
                    t0 = time.perf_counter()
                    for _ in range(args.iters):
                        call()
                    dt = (time.perf_counter() - t0) / args.iters
                    assert torch.equal(view, want), (storage, k, a, b, method)
                    n = want.numel() * want.element_size()
                    rows.append({"storage": storage, "tensor": list(t.shape), "columns": [a, b], "shape": label, "row_bytes": (b - a) * 2,
                                 "object_bytes": n, "method": method, "ms_per_call": round(dt * 1e3, 4),
                                 "delivered_GBps": round(n / dt / 1e9, 3)})
                del target, view
                store.remove([key])
        for r in rows:
            r.update({"gpu": name, "power_limit": power})
            print(json.dumps(r))
    finally:
        cl.stop()


if __name__ == "__main__":
    main()
