"""Packed (MXFP8) paged block puts and gets (TensorStore.put_blocks / get_blocks_into with pack_fp8=True, the paged
gathering load of the fused pack kernel and the paged scattering store of the fused unpack kernel) against the way a user
moves packed blocks of a paged KV cache without them, on one GPU.

    python bench/fp8_paged_bench.py [--iters 10] [--warmup 2]

A stacked bf16 KV cache [32, 2, 2048, 16, 8, 128] (32 KiB blocks, 4 GiB) with 256 random blocks selected along dim 2 is
one request's KV: one object of 16,384 pages, 512 MiB wide and 264 MiB packed.  Three more bf16 shapes cut the pages
smaller at the same block count: [32, 2, 2048, 8, 8, 128] (16 KiB), [.., 4, 8, 128] (8 KiB) and [.., 2, 8, 128] (4 KiB);
an fp16 cache [32, 2, 2048, 16, 8, 128] and an fp32 cache [32, 2, 2048, 8, 8, 128] have 32 KiB pages.  Each is moved
three ways:
  (a) paged fp8:    the paged packed calls put_blocks / get_blocks_into make at any page size
                    (FP8_PAGED_MIN_PAGE_BYTES = 0),
  (b) index_select: put(key, cache.index_select(2, ids), pack_fp8=True) / cache.index_copy_(2, new_ids, get(key)),
  (c) as shipped:   put_blocks(key, cache, ids, dim=2, pack_fp8=True) / get_blocks_into(key, cache, new_ids, dim=2),
                    which route pages below FP8_PAGED_MIN_PAGE_BYTES to (b).
For (a) it also reports the kernel time of the fused pack or unpack (CUDA events, fabric.last_device_ms), so the host
share of a call is visible.  Objects sit in this GPU's HBM slab (BBH64, the packed objects' digest).  For each it reports
ms per call (host clock around a call that ends in a device synchronise; min / median / max over the timed calls), wide
GB/s at the median, and the peak extra device memory the call allocated.  Each get is checked against index_copy_ of the
unpacked blocks.  Prints one JSON line per row with the card name and power limit read in the same run.
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
        sys.exit("fp8_paged_bench needs a GPU")
    name, power = card()
    cl = GpuRankCluster(slab_bytes=1280 * MiB, cluster_id="fp8-paged-bench")
    shipped = tensor_store.FP8_PAGED_MIN_PAGE_BYTES
    try:
        shapes = [("bf16 32 KiB pages", torch.bfloat16, (32, 2, 2048, 16, 8, 128)), ("bf16 16 KiB pages", torch.bfloat16, (32, 2, 2048, 8, 8, 128)),
                  ("bf16 8 KiB pages", torch.bfloat16, (32, 2, 2048, 4, 8, 128)), ("bf16 4 KiB pages", torch.bfloat16, (32, 2, 2048, 2, 8, 128)),
                  ("fp16 32 KiB pages", torch.float16, (32, 2, 2048, 16, 8, 128)), ("fp32 32 KiB pages", torch.float32, (32, 2, 2048, 8, 8, 128))]
        cfg = _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[_bb.StorageClass.RAM_GPU])
        store = TensorStore(cl.client, cfg)
        for label, dtype, shape in shapes:
            g = torch.Generator(device="cuda").manual_seed(5)
            cache = torch.randn(shape, device="cuda", generator=g).to(dtype)
            perm = torch.randperm(shape[2], generator=torch.Generator().manual_seed(6))
            ids, new_ids = perm[:256], perm[256:512]
            ids_d, new_d = ids.cuda(), new_ids.cuda()
            sel = cache.index_select(2, ids_d)
            nbytes = sel.numel() * sel.element_size()
            _, page, _ = TensorStore._block_pages(cache, 2, ids.numpy(), 0)
            store.put("ref", sel, pack_fp8=True)
            want = store.get("ref")  # the unpacked blocks every get must store
            store.remove(["ref"])

            def routed(min_page, call):
                def run():
                    tensor_store.FP8_PAGED_MIN_PAGE_BYTES = min_page
                    try:
                        call()
                    finally:
                        tensor_store.FP8_PAGED_MIN_PAGE_BYTES = shipped
                return run

            def put_b():
                store.put("b", cache.index_select(2, ids_d), pack_fp8=True)

            def get_b():
                cache.index_copy_(2, new_d, store.get("b"))

            methods = [("(a) paged fp8", routed(0, lambda: store.put_blocks("a", cache, ids, dim=2, pack_fp8=True)),
                        routed(0, lambda: store.get_blocks_into("a", cache, new_ids, dim=2)), "a"),
                       ("(b) index_select + put / get + index_copy_", put_b, get_b, "b"),
                       ("(c) put_blocks / get_blocks_into as shipped", lambda: store.put_blocks("c", cache, ids, dim=2, pack_fp8=True),
                        lambda: store.get_blocks_into("c", cache, new_ids, dim=2), "c")]
            for method, put, get, key in methods:
                for op, call in (("put", put), ("get", get)):
                    times, extra, dev = [], 0, []
                    for it in range(args.warmup + args.iters):
                        if op == "put":
                            store.remove([key])
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
                        got = cache.index_select(2, new_d)
                        assert torch.equal(got.view(torch.int16 if got.element_size() == 2 else torch.int32),
                                           want.view(torch.int16 if want.element_size() == 2 else torch.int32)), (label, method)
                    med = statistics.median(times)
                    row = {"shape": label, "dtype": str(dtype)[6:], "cache": list(shape), "page_bytes": page, "pages": 32 * 2 * 256,
                           "wide_bytes": nbytes, "packed_bytes": nbytes // sel.element_size() * 33 // 32, "method": method, "op": op,
                           "ms_min": round(min(times) * 1e3, 3), "ms_median": round(med * 1e3, 3), "ms_max": round(max(times) * 1e3, 3),
                           "wide_GBps": round(nbytes / med / 1e9, 2), "peak_extra_MiB": round(extra / MiB, 1),
                           "kernel_ms_median": round(statistics.median(dev), 3) if method.startswith("(a)") else None, "calls": args.iters,
                           "fp8_paged_min_page_bytes": shipped}
                    print(json.dumps(dict(row, gpu=name, power_limit=power)), flush=True)
                store.remove([key])
            del cache, sel, want
            torch.cuda.empty_cache()
    finally:
        cl.stop()


if __name__ == "__main__":
    main()
