"""MXFP8 packing of fp16 and fp32 tensors fused into the put and get kernels (`wide=`) against what a user writes without
it, a conversion to bf16 around the fused bf16 calls, on one GPU.

    python bench/fp8_wide_bench.py [--iters 5] [--warmup 1] [--objects 64] [--mib 64]

For each wide type (bf16 as the baseline, fp16, fp32) the batch is `--objects` tensors of `--mib` MiB of wide data each
(64 x 64 MiB by default), stored in this GPU's HBM slab, one copy.  Methods, one batched client call each:
  - put fused:       batch_put_device_fp8(..., wide=type), the pack reading the tensors once;
  - put via bf16:    t.to(torch.bfloat16) into a temporary, then batch_put_device_fp8 of the temporaries (fp16 / fp32);
  - get fused:       batch_get_device_fp8(..., wide=type) into tensors of the type;
  - get via bf16:    batch_get_device_fp8 into bf16 temporaries, then out.copy_(temporary) (fp16 / fp32).
Each call is timed by a host clock around the call and a device synchronise; a put's keys are removed after each timed
call, outside the clock.  Reports ms per call and GB/s of wide bytes (objects x MiB / time), with the card name and power
limit, one JSON line per (type, method).  After the timed calls the fused get's result is compared with the stand-alone
kernels' pack + unpack of the same tensors.
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
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--objects", type=int, default=64)
    ap.add_argument("--mib", type=int, default=64)
    args = ap.parse_args()

    import torch

    from blackbird_b200 import _bb
    from blackbird_b200.parallel import GpuRankCluster

    if not torch.cuda.is_available():
        sys.exit("fp8_wide_bench needs a GPU")
    name, power = card()
    types = {"bf16": (torch.bfloat16, _bb.MxWide.BF16), "fp16": (torch.float16, _bb.MxWide.F16), "fp32": (torch.float32, _bb.MxWide.F32)}
    # the largest packed batch is bf16 / fp16: objects * mib / 2 * 33/32 MiB
    cl = GpuRankCluster(slab_bytes=(args.objects * args.mib * MiB // 2) * 33 // 32 + 256 * MiB, cluster_id="fp8-wide-bench")
    cfg = _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[_bb.StorageClass.RAM_GPU])
    c = cl.client
    rows = []
    try:
        for label, (dt, wide) in types.items():
            es = torch.empty((), dtype=dt).element_size()
            n = args.mib * MiB // es
            g = torch.Generator(device="cuda").manual_seed(11)
            src = torch.randn(args.objects, n, device="cuda", generator=g).to(dt)
            out = torch.empty_like(src)
            keys = [f"{label}/{i}" for i in range(args.objects)]
            s = torch.cuda.current_stream().cuda_stream
            tmp = torch.empty(args.objects, n, dtype=torch.bfloat16, device="cuda") if label != "bf16" else None

            def check(ecs):
                assert all(e == _bb.ErrorCode.OK for e in ecs), ecs[:3]

            def put_fused():
                check(c.batch_put_device_fp8(keys, [t.data_ptr() for t in src], [n] * args.objects, cfg, s, wide=wide))

            def put_bf16():
                tmp.copy_(src)
                check(c.batch_put_device_fp8(keys, [t.data_ptr() for t in tmp], [n] * args.objects, cfg, s))

            def get_fused():
                check(c.batch_get_device_fp8(keys, [t.data_ptr() for t in out], [n] * args.objects, s, wide=wide))

            def get_bf16():
                check(c.batch_get_device_fp8(keys, [t.data_ptr() for t in tmp], [n] * args.objects, s))
                out.copy_(tmp)

            def timed(call, after=None):
                total = 0.0
                for i in range(args.warmup + args.iters):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    call()
                    torch.cuda.synchronize()
                    if i >= args.warmup:
                        total += time.perf_counter() - t0
                    if after:
                        after()
                return total / args.iters

            def remove():
                c.batch_remove(keys)

            methods = [("put fused", put_fused, remove)] + ([("put via bf16", put_bf16, remove)] if tmp is not None else [])
            for m, call, after in methods:
                rows.append((label, m, timed(call, after)))
            put_fused()
            methods = [("get fused", get_fused, None)] + ([("get via bf16", get_bf16, None)] if tmp is not None else [])
            for m, call, after in methods:
                rows.append((label, m, timed(call, after)))
            get_fused()
            torch.cuda.synchronize()
            # the fused get equals the stand-alone kernels' pack + unpack of the same tensors
            packed = torch.empty(_bb.mxfp8_packed_bytes(n), dtype=torch.uint8, device="cuda")
            ref = torch.empty(n, dtype=dt, device="cuda")
            for i in (0, args.objects - 1):
                _bb.mxfp8_pack(src[i].data_ptr(), n, packed.data_ptr(), s, wide=wide)
                _bb.mxfp8_unpack(packed.data_ptr(), n, ref.data_ptr(), s, wide=wide)
                torch.cuda.synchronize()
                assert torch.equal(ref.view(torch.uint8), out[i].view(torch.uint8)), (label, i)
            remove()
            del src, out, tmp
            torch.cuda.empty_cache()
        wide_bytes = args.objects * args.mib * MiB
        for label, m, dt in rows:
            print(json.dumps({"type": label, "method": m, "objects": args.objects, "wide_MiB_per_object": args.mib,
                              "ms_per_call": round(dt * 1e3, 3), "wide_GBps": round(wide_bytes / dt / 1e9, 1), "gpu": name,
                              "power_limit": power}))
    finally:
        cl.stop()


if __name__ == "__main__":
    main()
