"""Paged puts and gets of per-layer KV caches with block ids that stay on the device (TensorStore.put_layer_blocks /
get_layer_blocks_into: the transfer engine's resolve kernel builds the page table on the GPU) against the ways a user
moves the same blocks without it, on one GPU.

    python bench/layer_blocks_bench.py [--iters 10] [--warmup 2]

One request's KV is 256 blocks selected along dim 1 of 32 per-layer bf16 caches [2, 2048, h, 8, 128]; h = 16, 8, 4, 2
gives pages of 32, 16, 8 and 4 KiB (at 32 KiB the 512 MiB object of paged_bench.py, split across layers).  The layers are
the slices of one stacked cache [32, 2, 2048, h, 8, 128], so the stacked routes read the same memory.  Unpacked objects
carry XXH3 or no checksum; packed (MXFP8, BBH64) objects of bf16 caches at the same page sizes and of fp16 and fp32
caches with 32 KiB pages (fp32: h halved) are run too, (c) left out and partial gets of k = 16 and 256.  Puts, four ways:
  (a) put_layer_blocks(key, layers, ids)          CUDA int32 ids, the device route at every page size;
  (b) put_blocks(key, stacked, ids, dim=2)        the paged put of the stacked cache, host ids (a numpy table per call);
  (c) batch_put_blocks, one object per layer      host ids;
  (d) put(stack([l.index_select(1, ids)]))        a 512 MiB temporary at 32 KiB pages.
Gets, whole and partial (k = 16, 128, 256 of the stored blocks, into random free blocks), the mirrors: (a)
get_layer_blocks_into, (b) get_blocks_into on the stacked cache, (c) batch_get_blocks_into per layer (whole only), (d)
get + index_select + index_copy_ per layer.  Every result is checked against (d).

For each it reports ms per call (host clock around a call that ends in a device synchronise; min / median / max), and
the transfer kernel's time (CUDA events, fabric.last_device_ms) for the fused routes.  The resolve kernel is launched
inside the engine's call, between the copy of the descriptor table and the transfer kernel, where no caller can put CUDA
events around it; its own time is read with torch.profiler (CUPTI kernel records) in a separate pass, one put and one
get per page size, so that tracing does not slow the timed calls.  Prints one JSON line per row with the card name and power limit read in the same run.
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
L, B, K = 32, 2048, 256


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
    """Host times and transfer kernel times of the timed calls; `before` runs untimed ahead of each call."""
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


def resolve_ms(fn):
    """Device time of the resolve kernel (and of the transfer kernels) in one call of fn, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "bb_" in e.name:
            key = "resolve" if "resolve_blocks" in e.name else "transfer"
            out[key] = out.get(key, 0.0) + e.device_time / 1e3
    return out


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
        sys.exit("layer_blocks_bench needs a GPU")
    name, power = card()
    cl = GpuRankCluster(slab_bytes=2560 * MiB, cluster_id="layer-blocks-bench")
    # every route at every page size: the thresholds are what this measures
    for t in ("PAGED_MIN_PAGE_BYTES", "FP8_PAGED_MIN_PAGE_BYTES", "FP8_PARTIAL_MIN_PAGE_BYTES", "LAYER_BLOCKS_MIN_PAGE_BYTES",
              "FP8_LAYER_BLOCKS_MIN_PAGE_BYTES"):
        setattr(tensor_store, t, 0)

    def emit(row, times, dev=None):
        row.update(ms_min=round(min(times) * 1e3, 3), ms_median=round(statistics.median(times) * 1e3, 3), ms_max=round(max(times) * 1e3, 3),
                   kernel_ms_median=round(statistics.median(dev), 3) if dev else None, calls=args.iters, gpu=name, power_limit=power)
        print(json.dumps(row), flush=True)

    try:
        kinds = [(torch.bfloat16, "XXH3", False, (32, 16, 8, 4)), (torch.bfloat16, "NONE", False, (32, 16, 8, 4)),
                 (torch.bfloat16, "BBH64", True, (32, 16, 8, 4)), (torch.float16, "BBH64", True, (32,)), (torch.float32, "BBH64", True, (32,))]
        for dtype, algo, packed, pages in kinds:
            es = torch.empty((), dtype=dtype).element_size()
            bits = {2: torch.int16, 4: torch.int32}[es]
            for page_kib in pages:
                h = page_kib * 1024 // (8 * 128 * es)
                g = torch.Generator(device="cuda").manual_seed(5)
                stacked = torch.randn((L, 2, B, h, 8, 128), device="cuda", generator=g).to(dtype)
                layers = [stacked[l] for l in range(L)]
                perm = torch.randperm(B, generator=torch.Generator().manual_seed(6))
                ids_h, free = perm[:K], perm[K:]
                ids_d = ids_h.to(device="cuda", dtype=torch.int32)
                ids_l = ids_h.tolist()
                cfg = _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, checksum=getattr(_bb.ChecksumAlgo, algo),
                                       preferred_classes=[_bb.StorageClass.RAM_GPU])
                store = TensorStore(cl.client, cfg)
                base = {"dtype": str(dtype)[6:], "packed": packed, "page_KiB": page_kib, "checksum": algo, "wide_bytes": L * 2 * K * page_kib * 1024}
                lkeys = [f"l/{l}" for l in range(L)]
                puts = [("(a) put_layer_blocks, CUDA int32 ids", lambda: store.put_layer_blocks("a", layers, ids_d, dim=1, pack_fp8=packed), ["a"]),
                        ("(b) put_blocks of the stacked cache, host ids", lambda: store.put_blocks("b", stacked, ids_l, dim=2, pack_fp8=packed), ["b"])]
                if not packed:
                    puts.append(("(c) batch_put_blocks, one object per layer",
                                 lambda: store.batch_put_blocks(lkeys, layers, [ids_l] * L, dim=1), lkeys))
                puts.append(("(d) index_select + stack + put",
                             lambda: store.put("d", torch.stack([l.index_select(1, ids_d) for l in layers]), pack_fp8=packed), ["d"]))
                for method, call, keys in puts:
                    times, dev = timed(call, args, cl.fabric, before=lambda: store.remove(keys))
                    emit(dict(base, op="put", method=method), times, dev if not method.startswith("(d)") else None)
                want = store.get("d")  # what the index_select route stores, packed or not
                assert torch.equal(store.get("a").view(bits), want.view(bits)) and torch.equal(store.get("b").view(bits), want.view(bits))
                if not packed:
                    assert torch.equal(want, torch.stack([l.index_select(1, ids_d) for l in layers]))
                    assert all(torch.equal(t, want[l]) for l, t in enumerate(store.batch_get(lkeys)))
                if algo != "NONE":
                    store.remove(["a"])
                    prof = resolve_ms(lambda: store.put_layer_blocks("a", layers, ids_d, dim=1, pack_fp8=packed))
                    print(json.dumps(dict(base, op="put", method="(a) profiler", resolve_ms=round(prof.get("resolve", 0), 4),
                                          transfer_ms=round(prof.get("transfer", 0), 4), gpu=name, power_limit=power)), flush=True)
                rng = torch.Generator().manual_seed(7)
                for k in (None, 16, 128, 256) if not packed else (None, 16, 256):
                    n = K if k is None else k
                    sel = None if k is None else torch.randperm(K, generator=rng)[:k]
                    into = free[torch.randperm(free.numel(), generator=rng)[:n]]
                    into_d, into_l = into.to(device="cuda", dtype=torch.int32), into.tolist()
                    sel_d = None if sel is None else sel.to(device="cuda", dtype=torch.int32)
                    sel_l = None if sel is None else sel.tolist()
                    ref = stacked.clone()
                    src = want if sel is None else want.index_select(2, sel_d)
                    for l in range(L):
                        ref[l].index_copy_(1, into_d.long(), src[l])
                    outs = {m: stacked.clone() for m in "abcd"}
                    gets = [("(a) get_layer_blocks_into, CUDA int32 ids",
                             lambda: store.get_layer_blocks_into("a", list(outs["a"]), into_d, dim=1, blocks=sel_d)),
                            ("(b) get_blocks_into of the stacked cache, host ids",
                             lambda: store.get_blocks_into("a", outs["b"], into_l, dim=2, blocks=sel_l))]
                    if k is None and not packed:
                        gets.append(("(c) batch_get_blocks_into, one object per layer",
                                     lambda: store.batch_get_blocks_into(lkeys, list(outs["c"]), [into_l] * L, dim=1)))

                    def whole():
                        t = store.get("a")
                        if sel_d is not None:
                            t = t.index_select(2, sel_d)
                        for l in range(L):
                            outs["d"][l].index_copy_(1, into_d.long(), t[l])

                    gets.append(("(d) get + index_select + index_copy_", whole))
                    for method, call in gets:
                        times, dev = timed(call, args, cl.fabric)
                        emit(dict(base, op="get" if k is None else "partial get", k=n, method=method), times,
                             dev if not method.startswith("(d)") else None)
                        assert torch.equal(outs[method[1]].view(bits), ref.view(bits)), (dtype, page_kib, algo, k, method)
                    if algo != "NONE" and k in (None, 16):
                        prof = resolve_ms(lambda: store.get_layer_blocks_into("a", list(outs["a"]), into_d, dim=1, blocks=sel_d))
                        print(json.dumps(dict(base, op="get" if k is None else "partial get", k=n, method="(a) profiler",
                                              resolve_ms=round(prof.get("resolve", 0), 4), transfer_ms=round(prof.get("transfer", 0), 4),
                                              gpu=name, power_limit=power)), flush=True)
                    del outs, ref
                store.remove(["a", "b", "d"] + lkeys)
                del stacked, layers, want
                torch.cuda.empty_cache()
    finally:
        cl.stop()


if __name__ == "__main__":
    main()
