"""Packed puts of sliced bf16 tensors (TensorStore.put(view, pack_fp8=True): the rows gathered by the fused pack kernel)
against a put of the slice made contiguous first, on one GPU.

    python bench/fp8_strided_put_bench.py [--iters 20] [--warmup 3]

Shapes: a [16384, 8192] bf16 weight (rows of 16 KiB) sliced along dim 1 at 1/2, 1/8 and 1/64 of a row (8 KiB, 2 KiB and
256 B per row); a KV layer [32768, 8, 128] sliced to 1 and 4 heads (256 B and 1 KiB per row; one head gives the
producer 128 row segments per 32 KiB bf16 tile, the most bulk loads per tile here); and t[::2] of a [16384, 8192]
tensor (16 KiB rows).  Each slice is stored as MXFP8 into this GPU's HBM slab (BBH64, one copy).  For each shape it
reports the time per call (host clock around a call that ends in a device synchronise), the bf16 GB/s (slice bytes /
time) and the peak memory torch allocated during the call beyond what was allocated before it, for
  - put(view):        TensorStore.put(view, pack_fp8=True) -- batch_put_device_fp8_strided, rows gathered while packing,
  - put(contiguous):  TensorStore.put(view.contiguous(), pack_fp8=True) -- a device copy into a temporary, then the fused
                      packed put.
The key is removed between calls, so every call allocates and writes a fresh object.  After the timed calls a get of
each key is compared bit for bit with a get of the other method's object.  Prints one JSON line per row with the card
name and power limit beside them.
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

    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    if not torch.cuda.is_available():
        sys.exit("fp8_strided_put_bench needs a GPU")
    name, power = card()
    cl = GpuRankCluster(slab_bytes=3 * 128 * MiB, cluster_id="fp8-strided-put-bench")
    try:
        store = TensorStore(cl.client)
        g = torch.Generator(device="cuda").manual_seed(3)
        w = torch.randn(16384, 8192, device="cuda", generator=g).to(torch.bfloat16)
        kv = torch.randn(32768, 8, 128, device="cuda", generator=g).to(torch.bfloat16)
        shapes = [("W[:, 0:4096]", "1/2 row", w[:, 0:4096]), ("W[:, 1024:2048]", "1/8 row", w[:, 1024:2048]),
                  ("W[:, 4096:4224]", "1/64 row", w[:, 4096:4224]), ("kv[:, 0:1, :]", "1 of 8 heads", kv[:, 0:1, :]),
                  ("kv[:, 2:6, :]", "4 of 8 heads", kv[:, 2:6, :]), ("W[::2]", "every other row", w[::2])]
        rows = []
        for label, what, view in shapes:
            r = store._gatherable(view)
            assert r is not None and store._fused_fp8_ok(view, store.config), label
            keys = {}
            for method, make in (("put(view)", lambda: view), ("put(contiguous)", lambda: view.contiguous())):
                key = f"{label}/{method}"
                keys[method] = key

                def call():
                    store.remove([key])
                    store.put(key, make(), pack_fp8=True)
                    torch.cuda.synchronize()

                for _ in range(args.warmup):
                    call()
                t0 = time.perf_counter()
                for _ in range(args.iters):
                    call()
                dt = (time.perf_counter() - t0) / args.iters
                store.remove([key])
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                store.put(key, make(), pack_fp8=True)
                torch.cuda.synchronize()
                peak = torch.cuda.max_memory_allocated() - base
                n = view.numel() * view.element_size()
                rows.append({"slice": label, "shape": what, "tensor": list(view.shape), "row_bytes": r[0], "bf16_bytes": n,
                             "method": method, "ms_per_call": round(dt * 1e3, 4), "bf16_GBps": round(n / dt / 1e9, 3),
                             "peak_alloc_MiB": round(peak / MiB, 3)})
            a, b = store.get(keys["put(view)"]), store.get(keys["put(contiguous)"])
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), label
            store.remove(list(keys.values()))
        for r in rows:
            r.update({"gpu": name, "power_limit": power})
            print(json.dumps(r))
    finally:
        cl.stop()


if __name__ == "__main__":
    main()
