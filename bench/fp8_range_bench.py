"""Row-range reads of an MXFP8-packed tensor: the fused element-range get against a whole get followed by a slice, on one GPU.

    python bench/fp8_range_bench.py [--iters 20] [--warmup 3]

One bf16 tensor of 8192 x 65536 elements (512 Mi elements, 1 GiB of bf16) is stored packed (`pack_fp8=True`, about
0.52 GiB in this GPU's HBM slab).  For windows of 1 row, 1 %, 10 % and 100 % of the rows it reports, per method:
  - fused-range: TensorStore.get_rows -- the whole packed object is read and verified, only the window is unpacked and
    stored into a window-sized result;
  - whole+slice: TensorStore.get of the whole tensor, then `[a:b].clone()` (what get_rows did for packed tensors before
    the fused range get);
the time per call (host clock around a call that ends in a device synchronise), the peak extra device memory of one call
(`torch.cuda.max_memory_allocated` above what was allocated before it, the result included) and the HBM bytes moved,
computed from the shapes: packed bytes read, bf16 bytes written, and for whole+slice the bf16 tensor written whole and
the slice read and written again.  Prints one JSON line per row, with the card name and power limit beside it.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

ROWS, COLS = 8192, 65536


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
    args = ap.parse_args()

    import torch

    from blackbird_b200 import _bb
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    if not torch.cuda.is_available():
        sys.exit("fp8_range_bench needs a GPU")
    name, power = card()
    n = ROWS * COLS
    packed_bytes = _bb.mxfp8_packed_bytes(n)
    cl = GpuRankCluster(slab_bytes=2 << 30, cluster_id="fp8-range-bench")
    try:
        store = TensorStore(cl.client)
        x = torch.empty(ROWS, COLS, dtype=torch.bfloat16, device="cuda")
        for r0 in range(0, ROWS, 1024):  # in slices: no 2 GiB fp32 temporary
            x[r0:r0 + 1024] = (torch.randn(1024, COLS, device="cuda") * 3).to(torch.bfloat16)
        store.put("fr/kv", x, pack_fp8=True)
        del x
        torch.cuda.empty_cache()
        rows = []
        for label, nrows in (("1 row", 1), ("1 %", ROWS // 100), ("10 %", ROWS // 10), ("100 %", ROWS)):
            a = (ROWS - nrows) // 2
            b = a + nrows
            w = nrows * COLS  # window elements

            def fused():
                return store.get_rows("fr/kv", a, b)

            def whole_slice():
                return store.get("fr/kv")[a:b].clone()

            ref = None
            for method, fn, moved in (("fused-range", fused, packed_bytes + 2 * w),
                                      ("whole+slice", whole_slice, packed_bytes + 2 * n + 4 * w)):
                for _ in range(args.warmup):
                    fn()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(args.iters):
                    out = fn()
                    torch.cuda.synchronize()
                dt = (time.perf_counter() - t0) / args.iters
                del out
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                out = fn()
                torch.cuda.synchronize()
                peak = torch.cuda.max_memory_allocated() - base
                if ref is None:
                    ref = out
                else:
                    assert torch.equal(out.view(torch.int16), ref.view(torch.int16)), "fused range differs from whole+slice"
                del out
                rows.append({"window": label, "rows": nrows, "window_elems": w, "method": method, "ms_per_call": round(dt * 1e3, 4),
                             "peak_extra_MiB": round(peak / (1 << 20), 2), "hbm_bytes_moved": moved,
                             "hbm_GiB_moved": round(moved / (1 << 30), 3)})
            del ref
        for r in rows:
            r.update({"gpu": name, "power_limit": power, "tensor_elems": n, "packed_bytes": packed_bytes})
            print(json.dumps(r))
    finally:
        cl.stop()


if __name__ == "__main__":
    main()
