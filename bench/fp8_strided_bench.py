"""Slices along an inner dimension of MXFP8-packed tensors: the fused strided get against a whole get followed by
`narrow().contiguous()`, on one GPU.

    python bench/fp8_strided_bench.py [--iters 20] [--warmup 3]

Two bf16 tensors of 32 Mi elements each are stored packed (`pack_fp8=True`, about 33 MiB each in this GPU's HBM slab):
  - a K layer of a KV cache, [32768 tokens, 8 heads, 128], sliced along the heads: 1, 2 and 4 of the 8 heads (rows of
    128 to 512 elements every 1024 elements);
  - the same layer heads-major, [8, 32768, 128], sliced along the tokens: tokens [0, 4096) of every head (8 rows of
    512 Ki elements every 4 Mi elements, a pitch far above 32 KiB).
Per slice and method:
  - fused-strided: TensorStore.get_slice -- the whole packed object is read and verified, only the slice's rows are
    unpacked and stored, densely, into a slice-sized result;
  - whole+narrow: TensorStore.get of the whole tensor, then `.narrow(dim, a, b - a).contiguous()` (what get_slice did for
    packed tensors before the fused strided get);
the time per call (host clock around a call that ends in a device synchronise), the peak extra device memory of one call
(`torch.cuda.max_memory_allocated` above what was allocated before it, the result included) and the HBM bytes read and
written per call, computed from the shapes: the packed object read and the slice written, and for whole+narrow also the
whole bf16 tensor written and the slice read again.  The two methods' results are compared bit for bit.  Prints one JSON
line per row, with the card name and power limit read in the same run.
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

TOKENS, HEADS, DIM = 32768, 8, 128


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
        sys.exit("fp8_strided_bench needs a GPU")
    name, power = card()
    n = TOKENS * HEADS * DIM
    packed_bytes = _bb.mxfp8_packed_bytes(n)
    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id="fp8-strided-bench")
    try:
        store = TensorStore(cl.client)
        k = (torch.randn(TOKENS, HEADS, DIM, device="cuda") * 3).to(torch.bfloat16)
        store.put("fs/k", k, pack_fp8=True)
        store.put("fs/k_heads_major", k.transpose(0, 1).contiguous(), pack_fp8=True)
        del k
        torch.cuda.empty_cache()
        # (label, key, dim, start, stop)
        slices = [("1 of 8 heads", "fs/k", 1, 3, 4), ("2 of 8 heads", "fs/k", 1, 2, 4), ("4 of 8 heads", "fs/k", 1, 4, 8),
                  ("tokens 0:4096 of every head", "fs/k_heads_major", 1, 0, 4096)]
        rows = []
        for label, key, dim, a, b in slices:
            shape = [TOKENS, HEADS, DIM] if key == "fs/k" else [HEADS, TOKENS, DIM]
            inner = 1
            for s in shape[dim + 1:]:
                inner *= s
            w = n // shape[dim] * (b - a)  # slice elements
            pitch_bytes = 2 * shape[dim] * inner

            def fused():
                return store.get_slice(key, dim, a, b)

            def whole_narrow():
                return store.get(key).narrow(dim, a, b - a).contiguous()

            ref = None
            for method, fn, read, written in (("fused-strided", fused, packed_bytes, 2 * w),
                                              ("whole+narrow", whole_narrow, packed_bytes + 2 * w, 2 * n + 2 * w)):
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
                    assert torch.equal(out.view(torch.int16), ref.view(torch.int16)), "fused strided differs from whole+narrow"
                del out
                rows.append({"slice": label, "dim": dim, "start": a, "stop": b, "slice_elems": w, "pitch_bytes": pitch_bytes,
                             "method": method, "ms_per_call": round(dt * 1e3, 4), "peak_extra_MiB": round(peak / (1 << 20), 2),
                             "hbm_bytes_read": read, "hbm_bytes_written": written,
                             "hbm_MiB_moved": round((read + written) / (1 << 20), 2)})
            del ref
        for r in rows:
            r.update({"gpu": name, "power_limit": power, "tensor_elems": n, "packed_bytes": packed_bytes})
            print(json.dumps(r))
    finally:
        cl.stop()


if __name__ == "__main__":
    main()
