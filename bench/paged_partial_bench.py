"""Partial restores of paged objects (TensorStore.get_blocks_into with `blocks`: a page table over the whole stored object
whose unselected pages are null, taken by the paged scattering store of bb_xfer or of the fused unpack) against the way a
user restores some stored blocks without it, on one GPU.

    python bench/paged_partial_bench.py [--iters 10] [--warmup 2]

One request's KV is 256 blocks of a stacked KV cache [32, 2, 2048, h, 8, 128] selected along dim 2 and stored as one
object with put_blocks, the workload of paged_bench.py: bf16 with h = 16, 8, 4, 2 gives pages of 32, 16, 8 and 4 KiB
(a 512 MiB object at 32 KiB).  Unpacked objects are stored with XXH3 and with no checksum; packed (MXFP8) objects of
bf16, fp16 and fp32 caches with the same page sizes (fp32: h halved) carry BBH64, the packed objects' digest.  From each,
k = 16, 128 and 256 stored blocks -- a prefix, and a random subset -- are restored into random free blocks of the cache,
two ways:
  (a) partial:  get_blocks_into(key, cache, ids, dim=2, blocks=sel) on the paged route at every page size
                (the page thresholds of tensor_store set to 0): the whole object is read and verified, only the
                selected pages are stored, no temporary;
  (b) get:      cache.index_copy_(2, ids, get(key).index_select(2, sel)), a whole-object temporary and two more passes.
For each it reports ms per call (host clock around a call that ends in a device synchronise; min / median / max over the
timed calls), and for (a) the kernel time of the transfer (CUDA events, fabric.last_device_ms).  Every restore is checked
against (b).  Prints one JSON line per row with the card name and power limit read in the same run.
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
        sys.exit("paged_partial_bench needs a GPU")
    name, power = card()
    cl = GpuRankCluster(slab_bytes=1280 * MiB, cluster_id="paged-partial-bench")
    # the paged route at every page size: the thresholds are what this measures
    tensor_store.PAGED_MIN_PAGE_BYTES = 0
    tensor_store.FP8_PAGED_MIN_PAGE_BYTES = 0
    tensor_store.FP8_PARTIAL_MIN_PAGE_BYTES = 0
    try:
        kinds = [("unpacked", torch.bfloat16, "XXH3"), ("unpacked", torch.bfloat16, "NONE"), ("packed", torch.bfloat16, "BBH64"),
                 ("packed", torch.float16, "BBH64"), ("packed", torch.float32, "BBH64")]
        for kind, dtype, algo in kinds:
            es = torch.empty((), dtype=dtype).element_size()
            cfg = _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, checksum=getattr(_bb.ChecksumAlgo, algo),
                                   preferred_classes=[_bb.StorageClass.RAM_GPU])
            store = TensorStore(cl.client, cfg)
            for page_kib in (32, 16, 8, 4):
                h = page_kib * 1024 // (8 * 128 * es)
                shape = (32, 2, 2048, h, 8, 128)
                g = torch.Generator(device="cuda").manual_seed(5)
                cache = torch.randn(shape, device="cuda", generator=g).to(dtype)
                perm = torch.randperm(shape[2], generator=torch.Generator().manual_seed(6))
                stored_ids, free = perm[:256], perm[256:]
                store.put_blocks("a", cache, stored_ids, dim=2, pack_fp8=kind == "packed")
                nbytes = 32 * 2 * 256 * page_kib * 1024
                rng = torch.Generator().manual_seed(7)
                for k in (16, 128, 256):
                    for sel_kind in ("prefix", "random"):
                        sel = torch.arange(k) if sel_kind == "prefix" else torch.randperm(256, generator=rng)[:k]
                        ids = free[torch.randperm(free.numel(), generator=rng)[:k]]
                        sel_d, ids_d = sel.cuda(), ids.cuda()
                        sel_l, ids_l = sel.tolist(), ids.tolist()
                        ref = cache.clone()

                        def partial():
                            store.get_blocks_into("a", cache, ids_l, dim=2, blocks=sel_l)

                        def whole():
                            ref.index_copy_(2, ids_d, store.get("a").index_select(2, sel_d))

                        for method, call in (("(a) partial get_blocks_into", partial), ("(b) get + index_select + index_copy_", whole)):
                            times, dev = [], []
                            for it in range(args.warmup + args.iters):
                                torch.cuda.synchronize()
                                t0 = time.perf_counter()
                                call()
                                torch.cuda.synchronize()
                                dt = time.perf_counter() - t0
                                if it >= args.warmup:
                                    times.append(dt)
                                    dev.append(cl.fabric.last_device_ms)
                            med = statistics.median(times)
                            row = {"kind": kind, "dtype": str(dtype)[6:], "checksum": algo, "page_KiB": page_kib, "wide_bytes": nbytes,
                                   "k": k, "selection": sel_kind, "method": method, "ms_min": round(min(times) * 1e3, 3),
                                   "ms_median": round(med * 1e3, 3), "ms_max": round(max(times) * 1e3, 3),
                                   "kernel_ms_median": round(statistics.median(dev), 3) if method.startswith("(a)") else None, "calls": args.iters}
                            print(json.dumps(dict(row, gpu=name, power_limit=power)), flush=True)
                        bits = {2: torch.int16, 4: torch.int32}[es]
                        assert torch.equal(cache.view(bits), ref.view(bits)), (kind, dtype, page_kib, k, sel_kind)
                store.remove(["a"])
                del cache, ref
                torch.cuda.empty_cache()
    finally:
        cl.stop()


if __name__ == "__main__":
    main()
