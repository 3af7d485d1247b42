"""Paged block puts and gets (TensorStore.put_blocks / get_blocks_into, the paged gathering load and scattering store of
the fused kernel) against the two ways a user moves the blocks of a paged KV cache without them, on one GPU.

    python bench/paged_bench.py [--iters 10] [--warmup 2]

A stacked bf16 KV cache [32, 2, 2048, 16, 8, 128] (32 KiB blocks, 4 GiB) with 256 random blocks selected along dim 2 is
one request's KV: one 512 MiB object of 16,384 pages.  Two more shapes cut the pages smaller at the same block count:
[32, 2, 2048, 8, 8, 128] (16 KiB), [32, 2, 2048, 4, 8, 128] (8 KiB), [32, 2, 2048, 16, 128] (4 KiB pages, 64 MiB) and
[32, 2, 2048, 2, 128] (512 B pages, 8 MiB).  Each is moved up to four ways:
  (a) paged:        the paged calls put_blocks / get_blocks_into make at any page size (PAGED_MIN_PAGE_BYTES = 0),
  (b) index_select: put(key, cache.index_select(2, ids)) / cache.index_copy_(2, new_ids, get(key)),
  (c) per page:     one object per page through batch_put_device / batch_get_device (32 KiB pages only),
  (d) put_blocks:   put_blocks(key, cache, ids, dim=2) / get_blocks_into(key, cache, new_ids, dim=2) as shipped, which
                    route pages below PAGED_MIN_PAGE_BYTES to (b).
For (a) it also reports the kernel time of the transfer (CUDA events, fabric.last_device_ms), so the host share of a
call is visible.
Objects sit in this GPU's HBM slab, with XXH3 and with no checksum.  For each it reports ms per call (host clock around a
call that ends in a device synchronise; min / median / max over the timed calls), payload GB/s at the median, and the
peak extra device memory the call allocated.  Each get is checked against index_copy_ of the selected blocks.  Prints one
JSON line per row with the card name and power limit read in the same run.
"""
import argparse
import json
import os
import statistics
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
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import torch

    from blackbird_b200 import _bb
    from blackbird_b200.ops import tensor_store
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    if not torch.cuda.is_available():
        sys.exit("paged_bench needs a GPU")
    name, power = card()
    cl = GpuRankCluster(slab_bytes=1280 * MiB, cluster_id="paged-bench")
    rows = []
    try:
        shapes = [("32 KiB pages", (32, 2, 2048, 16, 8, 128)), ("16 KiB pages", (32, 2, 2048, 8, 8, 128)), ("8 KiB pages", (32, 2, 2048, 4, 8, 128)),
                  ("4 KiB pages", (32, 2, 2048, 16, 128)), ("512 B pages", (32, 2, 2048, 2, 128))]
        shipped = tensor_store.PAGED_MIN_PAGE_BYTES
        for label, shape in shapes:
            g = torch.Generator(device="cuda").manual_seed(5)
            cache = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
            perm = torch.randperm(shape[2], generator=torch.Generator().manual_seed(6))
            ids, new_ids = perm[:256], perm[256:512]
            ids_d, new_d = ids.cuda(), new_ids.cuda()
            sel = cache.index_select(2, ids_d)
            nbytes = sel.numel() * sel.element_size()
            for algo in ("XXH3", "NONE"):
                cfg = _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, checksum=getattr(_bb.ChecksumAlgo, algo),
                                       preferred_classes=[_bb.StorageClass.RAM_GPU])
                store = TensorStore(cl.client, cfg)
                tensor_store.PAGED_MIN_PAGE_BYTES = 0
                src_pages, page, _ = TensorStore._block_pages(cache, 2, ids.numpy())
                dst_pages, _, _ = TensorStore._block_pages(cache, 2, new_ids.numpy())
                page_keys = [f"pp/{k}" for k in range(src_pages.size)]
                src_list, dst_list = src_pages.tolist(), dst_pages.tolist()
                tensor_store.PAGED_MIN_PAGE_BYTES = shipped

                def routed(min_page, call):
                    def run():
                        tensor_store.PAGED_MIN_PAGE_BYTES = min_page
                        call()
                    return run

                put_a = routed(0, lambda: store.put_blocks("a", cache, ids, dim=2))
                get_a = routed(0, lambda: store.get_blocks_into("a", cache, new_ids, dim=2))
                put_d = routed(shipped, lambda: store.put_blocks("a", cache, ids, dim=2))
                get_d = routed(shipped, lambda: store.get_blocks_into("a", cache, new_ids, dim=2))

                def put_b():
                    store.put("b", cache.index_select(2, ids_d))

                def get_b():
                    cache.index_copy_(2, new_d, store.get("b"))

                def put_c():
                    ecs = cl.client.batch_put_device(page_keys, src_list, [page] * len(page_keys), cfg, store._stream())
                    assert all(e == _bb.ErrorCode.OK for e in ecs)

                def get_c():
                    ecs, _ = cl.client.batch_get_device(page_keys, dst_list, [page] * len(page_keys), store._stream())
                    assert all(e == _bb.ErrorCode.OK for e in ecs)

                def remove_a():
                    store.remove(["a"])

                def remove_b():
                    store.remove(["b"])

                def remove_c():
                    cl.client.batch_remove(page_keys)

                methods = [("(a) paged calls", put_a, get_a, remove_a), ("(b) index_select + put / get + index_copy_", put_b, get_b, remove_b),
                           ("(d) put_blocks / get_blocks_into as shipped", put_d, get_d, remove_a)]
                if page == 32768:
                    methods.append(("(c) one object per page", put_c, get_c, remove_c))
                for method, put, get, remove in methods:
                    for op, call in (("put", put), ("get", get)):
                        times, extra, dev = [], 0, []
                        iters = min(args.iters, 3) if method.startswith("(c)") else args.iters
                        for it in range(args.warmup + iters):
                            if op == "put":
                                remove()
                            torch.cuda.synchronize()
                            base = torch.cuda.memory_allocated()
                            torch.cuda.reset_peak_memory_stats()
                            t0 = time.perf_counter()
                            call()
                            torch.cuda.synchronize()
                            dt = time.perf_counter() - t0
                            extra = max(extra, torch.cuda.max_memory_allocated() - base)
                            if it >= args.warmup:
                                times.append(dt)
                                dev.append(cl.fabric.last_device_ms)
                        if op == "get":
                            assert torch.equal(cache.index_select(2, new_d), sel), (label, algo, method)
                        med = statistics.median(times)
                        rows.append({"shape": label, "cache": list(shape), "page_bytes": page, "pages": src_pages.size, "object_bytes": nbytes,
                                     "checksum": algo, "method": method, "op": op, "ms_min": round(min(times) * 1e3, 3),
                                     "ms_median": round(med * 1e3, 3), "ms_max": round(max(times) * 1e3, 3),
                                     "payload_GBps": round(nbytes / med / 1e9, 2), "peak_extra_MiB": round(extra / MiB, 1),
                                     "kernel_ms_median": round(statistics.median(dev), 3) if method.startswith("(a)") else None, "calls": iters})
                        print(json.dumps(dict(rows[-1], gpu=name, power_limit=power)), flush=True)
                    remove()
            del cache, sel
            torch.cuda.empty_cache()
    finally:
        cl.stop()


if __name__ == "__main__":
    main()
