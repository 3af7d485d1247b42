"""Bundles (TensorStore.put_bundle / get_bundle_into, the segment-table gathering load and scattering store of the fused
kernel) against one object per tensor (batch_put / batch_get_into: N objects + N `#meta`), on one GPU.

    python bench/bundle_bench.py [--iters 10] [--warmup 2] [--rounds 2]

Workloads:
  (a) 4096 tensors of 4 KiB (16 MiB);
  (b) a synthetic bf16 transformer state_dict: 24 layers at hidden 2048 (qkv, o, up, gate, down projections and two
      norms and a qkv bias per layer, embeddings, an LM head and a final norm: 195 tensors, 3.5 GB);
  (c) (b) restored for a subset of 8 layers (get only: get_bundle_into naming those layers' tensors, against
      batch_get_into of those tensors).
Objects sit in this GPU's HBM slab, with XXH3 and with no checksum.  Each row reports ms per call (host clock around a
call that ends in a device synchronise; min / median / max over the timed calls of every round) and the objects the call
creates.  A separate pass reports the transfer kernel time of one segment put / get of (b) against a plain put / get of
one contiguous buffer of the same bytes, as [kernel ms from torch.profiler's CUPTI records, bb_xfer_kernel launches, the
engine's CUDA-event ms of its last batch].  Prints one JSON line per row with the card name and power limit
read in the same run.
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


def state_dict(torch, layers=24, hidden=2048, vocab=32000):
    sd, g = {}, torch.Generator(device="cuda").manual_seed(0)

    def t(*shape):
        return torch.randn(shape, generator=g, device="cuda", dtype=torch.bfloat16)

    sd["embed.weight"] = t(vocab, hidden)
    for i in range(layers):
        p = f"layers.{i}."
        sd[p + "attn_norm.weight"] = t(hidden)
        sd[p + "qkv.weight"], sd[p + "o.weight"] = t(3 * hidden, hidden), t(hidden, hidden)
        sd[p + "mlp_norm.weight"] = t(hidden)
        sd[p + "up.weight"], sd[p + "gate.weight"], sd[p + "down.weight"] = t(4 * hidden, hidden), t(4 * hidden, hidden), t(hidden, 4 * hidden)
        sd[p + "qkv.bias"] = t(3 * hidden)
    sd["norm.weight"] = t(hidden)
    sd["lm_head.weight"] = t(vocab, hidden)
    return sd


def kernel_ms(fn):
    """[transfer kernel ms, kernel launches] of one call of fn: the CUPTI records of bb_xfer_kernel, from torch.profiler
    in a session of its own."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ks = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "bb_xfer_kernel" in e.name]
    return [round(sum(e.device_time for e in ks) / 1e3, 3), len(ks)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()

    import torch

    from blackbird_b200 import _bb
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    name, power = card()
    cl = GpuRankCluster(slab_bytes=12 << 30, cluster_id="bundle-bench")

    def timed(fn, cleanup=None):
        out = []
        for r in range(args.rounds):
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

    def row(workload, algo, op, route, ms, objects, nbytes):
        print(json.dumps({"workload": workload, "checksum": algo, "op": op, "route": route, "ms_min": round(min(ms), 3),
                          "ms_median": round(statistics.median(ms), 3), "ms_max": round(max(ms), 3), "objects_per_call": objects,
                          "bytes": nbytes, "calls": len(ms), "card": name, "power_limit": power}), flush=True)

    try:
        small = {f"t{i}": torch.randint(0, 255, (4096,), dtype=torch.uint8, device="cuda") for i in range(4096)}
        sd = state_dict(torch)
        subset = {k: v for k, v in sd.items() if any(k.startswith(f"layers.{i}.") for i in range(8))}
        for algo in ("XXH3", "NONE"):
            cfg = _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, checksum=getattr(_bb.ChecksumAlgo, algo),
                                   preferred_classes=[_bb.StorageClass.RAM_GPU])
            store = TensorStore(cl.client, cfg)
            for wl, b in (("a:4096x4KiB", small), ("b:state_dict", sd)):
                nbytes = sum(t.numel() * t.element_size() for t in b.values())
                keys = [f"{wl}/{k}" for k in b]
                ms = timed(lambda: store.put_bundle(wl, b), lambda: store.remove([wl]))
                row(wl, algo, "put", "put_bundle", ms, 2, nbytes)
                ms = timed(lambda: store.batch_put(keys, list(b.values())), lambda: store.remove(keys))
                row(wl, algo, "put", "batch_put", ms, 2 * len(b), nbytes)
                store.put_bundle(wl, b)
                store.batch_put(keys, list(b.values()))
                outs = {k: torch.empty_like(v) for k, v in b.items()}
                ms = timed(lambda: store.get_bundle_into(wl, outs))
                assert all(torch.equal(outs[k], b[k]) for k in b)
                row(wl, algo, "get", "get_bundle_into", ms, 0, nbytes)
                ms = timed(lambda: store.batch_get_into(keys, list(outs.values())))
                row(wl, algo, "get", "batch_get_into", ms, 0, nbytes)
                if wl.startswith("b"):
                    sub = {k: torch.empty_like(v) for k, v in subset.items()}
                    nsub = sum(t.numel() * t.element_size() for t in sub.values())
                    ms = timed(lambda: store.get_bundle_into(wl, sub))
                    assert all(torch.equal(sub[k], subset[k]) for k in sub)
                    row("c:8-layer subset", algo, "get", "get_bundle_into", ms, 0, nsub)
                    skeys = [f"{wl}/{k}" for k in sub]
                    ms = timed(lambda: store.batch_get_into(skeys, list(sub.values())))
                    row("c:8-layer subset", algo, "get", "batch_get_into", ms, 0, nsub)
                    # transfer kernel time: a segment put / get of the state_dict against a plain one of the same bytes.
                    # The slab holds the bundle and the per-tensor objects until here; both go first, so that the two
                    # objects of this pass fit beside each other.
                    store.remove([wl] + keys)
                    flat = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
                    seg, plain = f"k/seg/{algo}", f"k/flat/{algo}"

                    def ok(what, ecs):
                        assert all(e == _bb.ErrorCode.OK for e in ecs), (what, ecs)

                    calls = (("segments put", lambda: store.put_bundle(seg, b)),
                             ("plain put", lambda: ok("plain put", cl.client.batch_put_device([plain], [flat.data_ptr()], [nbytes], cfg, 0))),
                             ("segments get", lambda: store.get_bundle_into(seg, outs)),
                             ("plain get", lambda: ok("plain get", cl.client.batch_get_device([plain], [flat.data_ptr()], [nbytes], 0)[0])))
                    kern = {label: kernel_ms(fn) + [round(cl.fabric.last_device_ms, 3)] for label, fn in calls}
                    print(json.dumps({"workload": wl, "checksum": algo, "kernel_ms": kern, "bytes": nbytes, "card": name, "power_limit": power}),
                          flush=True)
                    store.remove([seg])
                    ok("remove", cl.client.batch_remove([plain]))
                else:
                    store.remove([wl] + keys)
    finally:
        cl.stop()


if __name__ == "__main__":
    main()
