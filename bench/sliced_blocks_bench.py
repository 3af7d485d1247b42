"""Paged puts and gets of head-sliced KV blocks (TensorStore.put_blocks / get_blocks_into on a view such as
cache[:, :, :, h0:h1, :]: each block's page is rows inside the block) against the ways a user moves the same blocks
without the in-page row pattern, on one GPU.

    python bench/sliced_blocks_bench.py [--iters 20] [--warmup 3]

Workloads, 256 of 2048 blocks selected along the block dim:
  NHD  bf16 [2, 2048, 16, 32, 128], dim=1, slices of 1, 8 and 16 of the 32 heads (rows of 256, 2048 and 4096 bytes,
       16 rows per block and outer index);
  NHD  bf16 [2, 2048, 16, 32, 64], dim=1, a 1-head slice: rows of 128 bytes, below PAGED_MIN_ROW_BYTES, so that the
       benchmark has a workload on each side of that threshold;
  HND  bf16 [2048, 2, 32, 16, 128], dim=0, an 8-head slice: 2 rows of 32 KiB per block.
Each unpacked (XXH3) and packed (MXFP8, BBH64), put and get.  Routes:
  (a) the paged route with the row pattern  put_blocks / get_blocks_into of the view (thresholds set to 0);
  (b) index_select + put, get + index_copy_ (what TensorStore did for these views before);
  (c) a per-row page table through the byte paged calls (unpacked only): one page entry per row;
  (r) the paged route over a contiguous cache with pages of the same dense bytes (the kernel-time reference).
For each it reports ms per call (host clock around a call that ends in a device synchronise; min / median / max over
--iters calls) and, for the fused routes, the transfer kernel's median time (CUDA events, fabric.last_device_ms).
Every result is checked against (b).  One JSON line per row, with the card name and power limit read in the same run.
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
K = 256


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


def timed(call, args, fabric, before=None):
    import torch

    times, dev = [], []
    for it in range(args.warmup + args.iters):
        if before:
            before()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        call()
        torch.cuda.synchronize()
        if it >= args.warmup:
            times.append(time.perf_counter() - t0)
            dev.append(fabric.last_device_ms)
    return times, dev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import numpy as np
    import torch

    from blackbird_b200 import _bb
    from blackbird_b200.ops import tensor_store
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    if not torch.cuda.is_available():
        sys.exit("sliced_blocks_bench needs a GPU")
    name, power = card()
    cl = GpuRankCluster(slab_bytes=2048 * MiB, cluster_id="sliced-blocks-bench")
    for t in ("PAGED_MIN_PAGE_BYTES", "FP8_PAGED_MIN_PAGE_BYTES", "FP8_PARTIAL_MIN_PAGE_BYTES", "PAGED_MIN_ROW_BYTES"):
        setattr(tensor_store, t, 0)

    def emit(row, times, dev=None):
        row.update(ms_min=round(min(times) * 1e3, 3), ms_median=round(statistics.median(times) * 1e3, 3), ms_max=round(max(times) * 1e3, 3),
                   kernel_ms_median=round(statistics.median(dev), 3) if dev else None, calls=args.iters, gpu=name, power_limit=power)
        print(json.dumps(row), flush=True)

    # (layout, cache shape, block dim, head dim, heads sliced)
    loads = [("NHD", (2, 2048, 16, 32, 128), 1, 3, 1), ("NHD", (2, 2048, 16, 32, 128), 1, 3, 8), ("NHD", (2, 2048, 16, 32, 128), 1, 3, 16),
             ("NHD", (2, 2048, 16, 32, 64), 1, 3, 1), ("HND", (2048, 2, 32, 16, 128), 0, 2, 8)]
    try:
        for layout, shape, dim, hdim, nh in loads:
            g = torch.Generator(device="cuda").manual_seed(5)
            cache = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
            view = cache.narrow(hdim, 4, nh)
            perm = torch.randperm(shape[dim], generator=torch.Generator().manual_seed(6))
            ids_l, into_l = perm[:K].tolist(), perm[K:2 * K].tolist()
            ids_d, into_d = perm[:K].cuda(), perm[K:2 * K].cuda()
            pg = TensorStore._block_pages(view, dim, np.asarray(ids_l, dtype=np.int64), 0)
            row_w, row_p = pg[2]
            dense = view.index_select(dim, ids_d)
            # the contiguous reference: a cache whose blocks are exactly the slice's dense bytes
            ref_shape = list(view.shape)
            contig = torch.empty(ref_shape, dtype=torch.bfloat16, device="cuda").copy_(view)
            for packed in (False, True):
                algo = "BBH64" if packed else "XXH3"
                cfg = _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, checksum=getattr(_bb.ChecksumAlgo, algo),
                                       preferred_classes=[_bb.StorageClass.RAM_GPU])
                store = TensorStore(cl.client, cfg)
                base = {"layout": layout, "shape": list(shape), "heads": nh, "row_bytes": row_w, "row_pitch": row_p,
                        "rows_per_page": pg[1] // row_w, "page_bytes": pg[1], "packed": packed, "checksum": algo,
                        "object_bytes": dense.numel() * 2}
                puts = [("(a) paged rows", lambda: store.put_blocks("a", view, ids_l, dim=dim, pack_fp8=packed)),
                        ("(b) index_select + put", lambda: store.put("b", view.index_select(dim, ids_d), pack_fp8=packed)),
                        ("(r) contiguous paged", lambda: store.put_blocks("r", contig, ids_l, dim=dim, pack_fp8=packed))]
                if not packed:
                    rows_tab = [np.asarray([a + r * row_p for a in pg[0] for r in range(pg[1] // row_w)], dtype=np.int64)]

                    def per_row_put():
                        ecs = cl.client.batch_put_device_paged(["c"], rows_tab, [row_w], cfg, torch.cuda.current_stream().cuda_stream)
                        assert ecs == [_bb.ErrorCode.OK]
                        store._put_metas(["c"], [tensor_store._meta(torch.bfloat16, list(dense.shape), False)])

                    puts.append(("(c) per-row page table", per_row_put))
                for method, call in puts:
                    k = method[1]
                    times, dev = timed(call, args, cl.fabric, before=lambda: store.remove([k]))
                    emit(dict(base, op="put", method=method), times, dev if k != "b" else None)
                want = store.get("b")
                bits = torch.int16
                for k in ("a", "r") + (("c",) if not packed else ()):
                    assert torch.equal(store.get(k).view(bits), want.view(bits)), (layout, nh, packed, k)
                ref = cache.clone()
                ref.narrow(hdim, 4, nh).index_copy_(dim, into_d, want)
                outs = {m: cache.clone() for m in "abc"}
                rtab = None
                if not packed:
                    rt = TensorStore._block_pages(outs["c"].narrow(hdim, 4, nh), dim, np.asarray(into_l, dtype=np.int64), 0)
                    rtab = [np.asarray([a + r * row_p for a in rt[0] for r in range(rt[1] // row_w)], dtype=np.int64)]
                rcontig = contig.clone()

                def whole():
                    outs["b"].narrow(hdim, 4, nh).index_copy_(dim, into_d, store.get("a"))

                gets = [("(a) paged rows", lambda: store.get_blocks_into("a", outs["a"].narrow(hdim, 4, nh), into_l, dim=dim)),
                        ("(b) get + index_copy_", whole),
                        ("(r) contiguous paged", lambda: store.get_blocks_into("a", rcontig, into_l, dim=dim))]
                if not packed:
                    gets.append(("(c) per-row page table",
                                 lambda: cl.client.batch_get_device_paged(["a"], rtab, [row_w], torch.cuda.current_stream().cuda_stream)))
                for method, call in gets:
                    times, dev = timed(call, args, cl.fabric)
                    emit(dict(base, op="get", method=method), times, dev if method[1] != "b" else None)
                    if method[1] in "abc":
                        assert torch.equal(outs[method[1]].view(bits), ref.view(bits)), (layout, nh, packed, method)
                store.remove(["a", "b", "c", "r"])
                del outs, ref, rcontig
            del cache, view, contig, dense
            torch.cuda.empty_cache()
    finally:
        cl.stop()


if __name__ == "__main__":
    main()
