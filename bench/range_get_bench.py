"""Byte-range device gets against whole-object gets followed by a slice copy, on one GPU.

    python bench/range_get_bench.py [--iters 20] [--warmup 3]

256 MiB single-shard objects in this GPU's HBM slab, written with XXH3 and with no checksum; ranges of 4 KiB, 1 MiB and
64 MiB at an unaligned-to-tile, 16-byte aligned offset.  For each (algorithm, range size) it reports the time per call
(host clock around a call that ends in a stream synchronise) and the delivered GB/s (range bytes / time) of
  - range:       client.batch_get_device_range of the range,
  - whole+slice: client.batch_get_device of the whole object, then out.narrow(...).copy_() of the range,
and the p50 latency of single 4 KiB range gets.  A verified range read reads every overlapping shard whole (here: the
whole 256 MiB object); without a checksum only the range's tiles are read.  Prints one JSON line per row and the card
name and power limit beside them.
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
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--latency-iters", type=int, default=200)
    args = ap.parse_args()

    import torch

    from blackbird_b200 import _bb
    from blackbird_b200.parallel import GpuRankCluster

    if not torch.cuda.is_available():
        sys.exit("range_get_bench needs a GPU")
    name, power = card()
    size = 256 * MiB
    cl = GpuRankCluster(slab_bytes=3 * size, cluster_id="range-bench")
    try:
        s = torch.cuda.current_stream().cuda_stream
        src = torch.empty(size, dtype=torch.uint8, device="cuda")
        _bb.random_fill(src.data_ptr(), size, 7, s)
        whole = torch.empty(size, dtype=torch.uint8, device="cuda")
        rows = []
        for algo in ("XXH3", "NONE"):
            key = f"rb/{algo}"
            cfg = _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, checksum=getattr(_bb.ChecksumAlgo, algo),
                                   preferred_classes=[_bb.StorageClass.RAM_GPU])
            assert cl.client.batch_put_device([key], [src.data_ptr()], [size], cfg, s) == [_bb.ErrorCode.OK]
            for n in (4096, 1 * MiB, 64 * MiB):
                off = 3 * 16384 + 4096 + 16  # 16-byte aligned, inside a tile
                out = torch.empty(n, dtype=torch.uint8, device="cuda")

                def ranged():
                    ecs = cl.client.batch_get_device_range([key], [out.data_ptr()], [off], [n], s)
                    assert ecs == [_bb.ErrorCode.OK], ecs
                    torch.cuda.synchronize()

                def whole_slice():
                    ecs, _ = cl.client.batch_get_device([key], [whole.data_ptr()], [size], s)
                    assert ecs == [_bb.ErrorCode.OK], ecs
                    out.copy_(whole.narrow(0, off, n))
                    torch.cuda.synchronize()

                for label, fn in (("range", ranged), ("whole+slice", whole_slice)):
                    for _ in range(args.warmup):
                        fn()
                    t0 = time.perf_counter()
                    for _ in range(args.iters):
                        fn()
                    dt = (time.perf_counter() - t0) / args.iters
                    assert torch.equal(out, src[off:off + n])
                    rows.append({"algo": algo, "range_bytes": n, "method": label, "ms_per_call": round(dt * 1e3, 4),
                                 "delivered_GBps": round(n / dt / 1e9, 3)})
            # p50 of single 4 KiB range gets
            out = torch.empty(4096, dtype=torch.uint8, device="cuda")
            lat = []
            for i in range(args.warmup + args.latency_iters):
                t0 = time.perf_counter()
                ecs = cl.client.batch_get_device_range([key], [out.data_ptr()], [16 * (i % 1000)], [4096], s)
                torch.cuda.synchronize()
                if i >= args.warmup:
                    lat.append(time.perf_counter() - t0)
                assert ecs == [_bb.ErrorCode.OK]
            rows.append({"algo": algo, "range_bytes": 4096, "method": "range single-call p50", "p50_us": round(statistics.median(lat) * 1e6, 2)})
        for r in rows:
            r.update({"gpu": name, "power_limit": power, "object_bytes": size})
            print(json.dumps(r))
    finally:
        cl.stop()


if __name__ == "__main__":
    main()
