"""Slice gets into existing tensors (TensorStore.get_slice_into, stored by the windowed scattering store of the fused get
kernel) against what a user writes without it, get_slice into a fresh tensor and a copy into the view, on one GPU.

    python bench/slice_into_bench.py [--iters 30] [--warmup 3] [--rounds 3]

A [16384, 8192] bf16 weight (256 MiB) is stored whole, and a tensor-parallel rank loads a column shard of it into its
place in a fused parameter three times as wide ([16384, 3 * w]), for shards of 1/2, 1/8 and 1/64 of a row (8 KiB, 2 KiB
and 256 B per row); a [32, 64, 4096] bf16 KV layer (16 MiB) gives a head range kv[:, 16:48, :] into the same heads of a
live buffer.  Each tensor is stored in this GPU's HBM slab with XXH3, with no checksum, and packed as MXFP8.  Each
(storage, shape) is timed in `rounds` rounds that alternate the two methods:
  - slice_into:       TensorStore.get_slice_into(key, view, dim, a, b) -- one windowed scattering get,
  - get_slice + copy_: view.copy_(TensorStore.get_slice(key, dim, a, b)) -- a slice-sized temporary and a device copy,
reporting per round the time per call (host clock over `iters` calls, each of which returns once its get has finished
on the device, closed by a device synchronise) and the stream time per call (CUDA events around the same calls: the
span of the stream, host gaps between launches included), then min / median / max over the rounds.  After the timed
calls the view is compared with the stored tensor's slice and the fused parameter's other columns with their canary.

A second section times the transfer kernel alone (XferEngine device time, CUDA events around the launch) for window and
destination shapes that cut tiles into uneven pieces, on a 64 MiB object with XXH3: a few window rows per tile that each
land in one or two destination rows, a warp's worth of window rows per tile that each span 16 short destination rows,
and long window rows cut into 128 destination rows each.  Each is compared with the same window stored densely (the
strided get) and with a plain whole-object get, `iters` launches per round, min / median / max over the rounds.
Prints one JSON line per row with the card name and power limit beside them.
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


def spread(v):
    return {"min": round(min(v), 4), "median": round(statistics.median(v), 4), "max": round(max(v), 4)}


def kernel_rows(args, rows):
    """The kernel-only section (see the module docstring): rows of {shape, method, device_ms}."""
    import numpy as np
    import torch

    from blackbird_b200 import _bb

    eng = _bb.XferEngine(0, 64, 2)
    n = 64 * MiB
    src = torch.empty(n, dtype=torch.uint8, device="cuda")
    _bb.random_fill(src.data_ptr(), n, 5, torch.cuda.current_stream().cuda_stream)
    plain = torch.empty(n, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    (dg,), _, _ = eng.run([(src.data_ptr(), plain.data_ptr(), n)], _bb.ChecksumAlgo.XXH3, st)
    # (label, window width, window pitch, destination width, destination pitch), in bytes, from object offset 0
    shapes = [("8 window rows a tile, 1 piece each", 1024, 2048, 1024, 1536), ("8 window rows a tile, 1-2 pieces each", 1024, 2048, 768, 1024),
              ("31 window rows a tile, 16 pieces each", 512, 528, 32, 48), ("2 window rows a tile, 128 pieces each", 8192, 16384, 64, 96)]
    for label, w, p, dw, dp in shapes:
        r = (n - w) // p + 1
        total = r * w
        last = total - 1
        out = torch.empty((last // dw) * dp + last % dw + 1, dtype=torch.uint8, device="cuda")
        dense = torch.empty(total, dtype=torch.uint8, device="cuda")
        win = (0, (r - 1) * p + w, p, w, 0)
        items = {"window into rows": (src.data_ptr(), out.data_ptr(), n, dg, _bb.XFER_VERIFY, 0, win) + (None,) * 6 + ((dp, dw, 0),),
                 "strided get (dense)": (src.data_ptr(), dense.data_ptr(), n, dg, _bb.XFER_VERIFY, 0, win),
                 "whole get": (src.data_ptr(), plain.data_ptr(), n, dg, _bb.XFER_VERIFY)}
        per = {k: [] for k in items}
        for _ in range(args.rounds):
            for method, it in items.items():
                for _ in range(args.warmup):
                    eng.run([it], _bb.ChecksumAlgo.XXH3, st)
                ms = []
                for _ in range(args.iters):
                    _, status, dms = eng.run([it], _bb.ChecksumAlgo.XXH3, st)
                    assert status == [0], (label, method)
                    ms.append(dms)
                per[method].append(statistics.median(ms))
        torch.cuda.synchronize()
        got, ref = out.cpu().numpy(), dense.cpu().numpy()
        q = np.arange(total, dtype=np.int64)
        assert np.array_equal(got[(q // dw) * dp + q % dw], ref), label
        for method, v in per.items():
            rows.append({"section": "kernel", "shape": label, "object_bytes": n, "window": [w, p], "dst_rows": [dw, dp], "stored_bytes": total,
                         "method": method, "rounds": args.rounds, "iters": args.iters, "device_ms": spread(v)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch

    from blackbird_b200 import _bb
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    if not torch.cuda.is_available():
        sys.exit("slice_into_bench needs a GPU")
    name, power = card()
    cl = GpuRankCluster(slab_bytes=3 * 256 * MiB, cluster_id="slice-into-bench")
    try:
        g = torch.Generator(device="cuda").manual_seed(3)
        tensors = {"weight": torch.randn(16384, 8192, device="cuda", generator=g).to(torch.bfloat16),
                   "kv": torch.randn(32, 64, 4096, device="cuda", generator=g).to(torch.bfloat16)}
        # (tensor, dim, [a, b), label)
        shapes = [("weight", 1, 0, 4096, "TP shard 1/2 row"), ("weight", 1, 1024, 2048, "TP shard 1/8 row"),
                  ("weight", 1, 4096, 4224, "TP shard 1/64 row"), ("kv", 1, 16, 48, "heads 16:48")]
        rows = []
        for storage in ("XXH3", "NONE", "MXFP8"):
            algo = "BBH64" if storage == "MXFP8" else storage
            store = TensorStore(cl.client, _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0,
                                                            checksum=getattr(_bb.ChecksumAlgo, algo),
                                                            preferred_classes=[_bb.StorageClass.RAM_GPU]))
            for k, dim, a, b, label in shapes:
                t = tensors[k]
                key = f"{storage}/{k}"
                store.put(key, t, pack_fp8=storage == "MXFP8")
                want = store.get_slice(key, dim, a, b)
                if k == "weight":  # the fused parameter: the shard's columns at its place among 3 shards' worth
                    target = torch.full((t.shape[0], 3 * (b - a)), 7.0, device="cuda", dtype=t.dtype)
                    place = (b - a, 2 * (b - a))
                else:  # the same heads of a live buffer
                    target = torch.full_like(t, 7.0)
                    place = (a, b)
                view = target.narrow(dim, place[0], place[1] - place[0])
                assert store._source_rows(view) is not None, label
                canary = target.clone()
                canary.narrow(dim, place[0], place[1] - place[0]).copy_(want)

                def into():
                    store.get_slice_into(key, view, dim, a, b)

                def get_copy():
                    view.copy_(store.get_slice(key, dim, a, b))

                per = {"slice_into": ([], []), "get_slice + copy_": ([], [])}
                for _ in range(args.rounds):
                    for method, call in (("slice_into", into), ("get_slice + copy_", get_copy)):
                        for _ in range(args.warmup):
                            call()
                        torch.cuda.synchronize()
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        t0 = time.perf_counter()
                        e0.record()
                        for _ in range(args.iters):
                            call()
                        e1.record()
                        torch.cuda.synchronize()
                        per[method][0].append((time.perf_counter() - t0) / args.iters * 1e3)
                        per[method][1].append(e0.elapsed_time(e1) / args.iters)
                        assert torch.equal(view, want), (storage, label, method)
                assert torch.equal(target, canary), (storage, label)
                n = want.numel() * want.element_size()
                for method, (call_ms, dev_ms) in per.items():
                    rows.append({"storage": storage, "tensor": list(t.shape), "dim": dim, "range": [a, b], "shape": label, "slice_bytes": n,
                                 "method": method, "rounds": args.rounds, "iters": args.iters, "call_ms": spread(call_ms),
                                 "stream_ms": spread(dev_ms), "delivered_GBps_median": round(n / statistics.median(call_ms) / 1e6, 3)})
                del target, view, canary
                store.remove([key])
        kernel_rows(args, rows)
        for r in rows:
            r.update({"gpu": name, "power_limit": power})
            print(json.dumps(r))
    finally:
        cl.stop()


if __name__ == "__main__":
    main()
