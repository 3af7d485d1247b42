"""MXFP8-packed bundles (TensorStore.put_bundle(..., pack_fp8=True), the segment-table gathering load and scattering
store of the fused pack and unpack kernels) against plain bundles and against one packed object per tensor
(batch_put(..., pack_fp8=True) / batch_get_into: N objects + N `#meta`), on one GPU.

    python bench/fp8_bundle_bench.py [--iters 5] [--warmup 1] [--rounds 2]

Workloads:
  (b) a synthetic bf16 transformer state_dict (bench/bundle_bench.py's: 24 layers at hidden 2048, 195 tensors, 3.5 GB);
      put, get_bundle (per tensor: batch_get), get_bundle_into of every entry and of 8 layers' entries (per tensor:
      batch_get_into of those tensors);
  (a) 4096 bf16 tensors of 4 KiB (16 MiB), the same calls without the subset.
Objects sit in this GPU's HBM slab; packed objects carry BBH64 (the fused pack computes it), plain bundles XXH3.  Each
row reports ms per call (host clock around a call that ends in a device synchronise; min / median / max over the timed
calls of every round), the objects the call creates and the bytes stored.  A separate pass reports the kernel time of one
packed segment put / get of (b) against a packed put / get of one contiguous buffer of the same elements, as [fused
MXFP8 kernel ms from torch.profiler's CUPTI records, its launches, ms of the bb_xfer_kernel launches that hash the
scales].  Prints one JSON line per row with the card name and power limit read in the same run.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.dont_write_bytecode = True  # the tree may be read-only
sys.path.insert(0, os.path.join(ROOT, "bench"))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bundle_bench import card, state_dict  # noqa: E402


def kernel_ms(fn):
    """[bb_xfer_fp8_kernel ms, its launches, bb_xfer_kernel ms] of one call of fn, from torch.profiler in a session of
    its own."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    fp8 = [e for e in ev if "bb_xfer_fp8_kernel" in e.name]
    raw = [e for e in ev if "bb_xfer_kernel" in e.name]
    return [round(sum(e.device_time for e in fp8) / 1e3, 3), len(fp8), round(sum(e.device_time for e in raw) / 1e3, 3)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()

    import torch

    from blackbird_b200 import _bb
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    name, power = card()
    cl = GpuRankCluster(slab_bytes=12 << 30, cluster_id="fp8-bundle-bench")

    def timed(fn, cleanup=None):
        out = []
        for _ in range(args.rounds):
            for i in range(args.warmup + args.iters):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                dt = (time.perf_counter() - t0) * 1e3
                if cleanup:
                    cleanup()
                if i >= args.warmup:
                    out.append(dt)
        return out

    def row(workload, op, route, ms, objects, stored, nbytes):
        print(json.dumps({"workload": workload, "op": op, "route": route, "ms_min": round(min(ms), 3), "ms_median": round(statistics.median(ms), 3),
                          "ms_max": round(max(ms), 3), "objects_per_call": objects, "bytes_stored": stored, "bytes": nbytes, "calls": len(ms),
                          "card": name, "power_limit": power}), flush=True)

    def packed_bytes(n):
        return _bb.mxfp8_packed_bytes((n + 31) // 32 * 32)

    try:
        cfg = _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, checksum=_bb.ChecksumAlgo.XXH3,
                               preferred_classes=[_bb.StorageClass.RAM_GPU])
        store = TensorStore(cl.client, cfg)
        g = torch.Generator(device="cuda").manual_seed(1)
        small = {f"t{i}": torch.randn(2048, generator=g, device="cuda").to(torch.bfloat16) for i in range(4096)}
        sd = state_dict(torch)
        layers = tuple(f"layers.{i}." for i in range(8))
        for wl, b in (("b:state_dict", sd), ("a:4096x4KiB", small)):
            nbytes = sum(t.numel() * t.element_size() for t in b.values())
            keys = [f"{wl}/{k}" for k in b]
            pk, pl = wl + "/packed", wl + "/plain"
            routes = (("packed bundle", lambda: store.put_bundle(pk, b, pack_fp8=True), lambda: store.remove([pk]), 2,
                       sum(packed_bytes(t.numel()) for t in b.values())),
                      ("plain bundle", lambda: store.put_bundle(pl, b), lambda: store.remove([pl]), 2, nbytes),
                      ("packed per tensor", lambda: store.batch_put(keys, list(b.values()), pack_fp8=True), lambda: store.remove(keys),
                       2 * len(b), sum(packed_bytes(t.numel()) for t in b.values())))
            for route, put, rm, objs, _ in routes:
                row(wl, "put", route, timed(put, rm), objs, None, nbytes)
            for route, put, _, _, _ in routes:
                put()
            stored = {r[0]: r[4] for r in routes}
            stored["packed bundle"] = packed_bytes(store._metas([pk], bundle=True)[0]["numel"])
            stored["plain bundle"] = store._metas([pl], bundle=True)[0]["total"]
            ref = store.get_bundle(pl)
            got = store.get_bundle(pk)
            per = dict(zip(b, store.batch_get(keys)))
            assert all(torch.equal(got[k].view(torch.int16), per[k].view(torch.int16)) for k in b), "packed bundle != per-tensor packed"
            assert all(torch.equal(ref[k], b[k]) for k in b)
            del ref, got, per
            gets = (("packed bundle", lambda: store.get_bundle(pk), lambda o: store.get_bundle_into(pk, o)),
                    ("plain bundle", lambda: store.get_bundle(pl), lambda o: store.get_bundle_into(pl, o)),
                    ("packed per tensor", lambda: store.batch_get(keys),
                     lambda o: store.batch_get_into([f"{wl}/{k}" for k in o], list(o.values()))))
            outs = {k: torch.empty_like(v) for k, v in b.items()}
            sub = {k: torch.empty_like(v) for k, v in b.items() if k.startswith(layers)}
            nsub = sum(t.numel() * t.element_size() for t in sub.values())
            for route, whole, into in gets:
                row(wl, "get_bundle", route, timed(whole), 0, stored[route], nbytes)
                row(wl, "get_bundle_into", route, timed(lambda: into(outs)), 0, stored[route], nbytes)
                if sub:
                    row("b:8-layer subset", "get_bundle_into", route, timed(lambda: into(sub)), 0, stored[route], nsub)
            store.remove([pk, pl] + keys)
            if wl.startswith("b"):
                # kernel time: a packed segment put / get of the state_dict against a packed put / get of one contiguous
                # buffer of the same elements
                numel = sum(t.numel() for t in b.values())
                flat = torch.empty(numel, dtype=torch.bfloat16, device="cuda")
                seg, plain = "k/seg", "k/flat"

                def ok(what, ecs):
                    assert all(e == _bb.ErrorCode.OK for e in ecs), (what, ecs)

                calls = (("segments put", lambda: store.put_bundle(seg, b, pack_fp8=True)),
                         ("plain put", lambda: ok("plain put", cl.client.batch_put_device_fp8([plain], [flat.data_ptr()], [numel], cfg, 0))),
                         ("segments get", lambda: store.get_bundle_into(seg, outs)),
                         ("plain get", lambda: ok("plain get", cl.client.batch_get_device_fp8([plain], [flat.data_ptr()], [numel], 0))))
                kern = {label: kernel_ms(fn) for label, fn in calls}
                print(json.dumps({"workload": wl, "kernel_ms": kern, "elements": numel, "card": name, "power_limit": power}), flush=True)
                store.remove([seg])
                ok("remove", cl.client.batch_remove([plain]))
    finally:
        cl.stop()


if __name__ == "__main__":
    main()
