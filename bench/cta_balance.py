#!/usr/bin/env python3
"""Per-CTA balance of the fused transfer kernel at the bench.py shape: 64 x 64 MiB objects, XXH3, one put and one get,
one chunk per batch, local HBM.

For every grid in --ctas (0 = the default geometry, `_bb.xfer_geometry`) it runs one put and one get with the tile trace
on (every tile stamped: load issued, landed in shared memory, store issued, slot released), groups the stamps by CTA with
cta_tile_run's arithmetic (CTA c owns tiles [c * tpc, (c + 1) * tpc), tpc = ceil(tiles / grid)) and reports per direction:

  first_load_us / last_release_us  p0 / p50 / p100 over CTAs of each CTA's first load issue and last slot release, from
                                   the first load of the launch
  idle_onset_us                    when a CTA slot first goes idle for good: the first CTA to finish after the last CTA
                                   has started (no run is left for the slot it frees).  With one persistent CTA per SM
                                   that is simply the first CTA to finish.
  tail_us, tail_frac               last release - idle onset, and its share of the traced span
  final_wave_release_us            p0 / p50 / p100 of the last release of the CTAs still running at the idle onset
  steady_GBps, tail_GBps           payload rate (tiles released x 16 KiB) before and after the idle onset

Then, with the trace off, the kernel-only time of the put and of the get at every grid (device events around each
launch, the fabric's total_device_ms, median of --reps).  The tile trace costs a few global stores per tile, so the traced
span is a little longer than the untraced kernel time.  One JSON line on stdout (and --out): the card name and its power
limit are part of every number.

  python bench/cta_balance.py --ctas 0,128,132,264 --reps 9
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from blackbird_b200 import _bb  # noqa: E402
from blackbird_b200.parallel import GpuRankCluster  # noqa: E402

TILE = 16384


def pcts(x):
    return {"p0": round(float(np.min(x)), 1), "p50": round(float(np.percentile(x, 50)), 1), "p100": round(float(np.max(x)), 1)}


def per_cta(trace, grid):
    """Balance of one traced launch of `grid` CTAs (trace = [tile][4] globaltimer ns)."""
    t = np.asarray(trace, dtype=np.uint64).reshape(-1, 4).astype(np.int64)
    tiles = len(t)
    assert (t > 0).all(), "a tile of the launch has no stamp"
    tpc = (tiles + grid - 1) // grid
    cta = np.arange(tiles) // tpc
    ncta = int(cta[-1]) + 1
    t0 = t[:, 0].min()
    load = (t[:, 0] - t0) / 1e3
    rel = (t[:, 3] - t0) / 1e3
    first = np.full(ncta, np.inf)
    last = np.zeros(ncta)
    np.minimum.at(first, cta, load)
    np.maximum.at(last, cta, rel)
    span = float(last.max())
    onset = float(last[last >= first.max()].min())
    wave = last[last >= onset]
    tail = span - onset
    before = int((rel <= onset).sum())
    return {"grid": grid, "ctas_with_tiles": ncta, "tiles_per_cta": tpc, "traced_span_us": round(span, 1),
            "first_load_us": pcts(first), "last_release_us": pcts(last), "idle_onset_us": round(onset, 1),
            "tail_us": round(tail, 1), "tail_frac": round(tail / span, 4), "final_wave_ctas": int(len(wave)),
            "final_wave_release_us": pcts(wave),
            "steady_GBps": round(before * TILE / onset / 1e3, 1) if onset > 0 else None,
            "tail_GBps": round((tiles - before) * TILE / tail / 1e3, 1) if tail > 0 else None}


def card():
    r = {"name": torch.cuda.get_device_name(0), "sms": torch.cuda.get_device_properties(0).multi_processor_count}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        r["power_limit"], r["max_sm_clock"] = [s.strip() for s in q.stdout.strip().split(",")[:2]]
    except Exception as e:  # the numbers are still the card's; say why its limit is missing
        r["power_limit"] = f"unavailable ({e})"
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ctas", default="0,128,132,264", help="comma-separated grids; 0 = the default geometry")
    ap.add_argument("--objects", type=int, default=64)
    ap.add_argument("--object-mib", type=int, default=64)
    ap.add_argument("--reps", type=int, default=9, help="untraced put + get pairs per grid (median)")
    ap.add_argument("--no-trace", action="store_true", help="kernel-only times only")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    nobj, size = args.objects, args.object_mib << 20
    step = nobj * size
    tiles = nobj * ((size + TILE - 1) // TILE)
    cl = GpuRankCluster(slab_bytes=3 * step + (64 << 20), cluster_id="cta-balance")
    dev = torch.device("cuda", cl.local_rank)
    stream = torch.cuda.current_stream().cuda_stream
    src = torch.empty(step, dtype=torch.uint8, device=dev)
    _bb.random_fill(src.data_ptr(), step, 0xB200, stream)
    out = torch.empty_like(src)
    src_ptrs = [src.data_ptr() + i * size for i in range(nobj)]
    out_ptrs = [out.data_ptr() + i * size for i in range(nobj)]
    cfg = _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, preferred_node="gpu0", ttl_ms=0,
                           checksum=_bb.ChecksumAlgo.XXH3, preferred_classes=[_bb.StorageClass.RAM_GPU])
    cl.client.set_device_pipeline_chunks(1)
    OK = _bb.ErrorCode.OK
    n = [0]

    def put_get(trace=False):
        keys = [f"cb/{n[0]}/{j}" for j in range(nobj)]
        n[0] += 1
        cl.fabric.set_tile_trace(trace)
        m0 = cl.fabric.total_device_ms
        assert all(e == OK for e in cl.client.batch_put_device(keys, src_ptrs, [size] * nobj, cfg, stream))
        m1 = cl.fabric.total_device_ms
        tp = cl.fabric.tile_trace() if trace else None
        ecs, _ = cl.client.batch_get_device(keys, out_ptrs, [size] * nobj, stream)
        assert all(e == OK for e in ecs)
        m2 = cl.fabric.total_device_ms
        tg = cl.fabric.tile_trace() if trace else None
        assert all(e == OK for e in cl.client.batch_remove(keys))
        cl.fabric.set_tile_trace(False)
        return m1 - m0, m2 - m1, tp, tg

    res = {"card": card(), "shape": f"{nobj} x {args.object_mib} MiB, XXH3, one chunk", "tiles": tiles,
           "torch": torch.__version__, "grids": []}
    for g in [int(x) for x in args.ctas.split(",")]:
        cl.fabric.set_max_ctas(g)
        # builds older than the short-CTA geometry have no xfer_geometry: measure them at an explicit grid
        geo = _bb.xfer_geometry(_bb.ChecksumAlgo.XXH3, tiles, g) if hasattr(_bb, "xfer_geometry") else {"grid": g}
        row = {"ctas": g, "geometry": geo}
        for _ in range(2):
            put_get()
        torch.cuda.synchronize()
        assert torch.equal(src, out), "payload mismatch"
        times = [put_get()[:2] for _ in range(args.reps)]
        row["put_ms"] = round(float(np.median([t[0] for t in times])), 4)
        row["get_ms"] = round(float(np.median([t[1] for t in times])), 4)
        row["put_ms_range"] = [round(min(t[0] for t in times), 4), round(max(t[0] for t in times), 4)]
        row["get_ms_range"] = [round(min(t[1] for t in times), 4), round(max(t[1] for t in times), 4)]
        if not args.no_trace:
            _, _, tp, tg = put_get(trace=True)
            row["put"] = per_cta(tp, geo["grid"])
            row["get"] = per_cta(tg, geo["grid"])
        res["grids"].append(row)
    cl.fabric.set_max_ctas(0)
    cl.stop()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
