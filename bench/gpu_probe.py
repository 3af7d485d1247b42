#!/usr/bin/env python3
"""First-contact GPU diagnostics for the fused transfer kernel.

phase=probe : impulse probes through the wgmma int8 MMA (dumps the raw accumulators and
              derives which (row, k) the hardware assigns to each tile-linear byte offset),
              then digest / copy correctness against the CPU BBH64 model.
phase=perf  : single-GPU bandwidth of the fused kernel vs copy-only, SIMT copy, cudaMemcpy.
Prints to stdout.
"""
import argparse
import sys
import time
import traceback

import numpy as np
import torch

sys.path.insert(0, ".")
from blackbird_b200 import _bb  # noqa: E402

T = _bb.TILE_BYTES


def stream():
    return torch.cuda.current_stream().cuda_stream


def phase_probe():
    dev = torch.device("cuda:0")
    eng = _bb.XferEngine(0, 4096, 2)
    print("smem bytes", _bb.xfer_smem_bytes())
    # ---- impulse probes
    offsets = [0, 1, 15, 16, 17, 31, 32, 112, 127, 128, 129, 255, 256, 1023, 1024, 1025, 2048, 4096, 8191, 8192, 16383]
    ok_all = True
    for o in offsets:
        src = torch.zeros(T, dtype=torch.uint8, device=dev)
        src[o] = 1
        dst = torch.zeros(T, dtype=torch.uint8, device=dev)
        dg, st, ms = eng.run([(src.data_ptr(), dst.data_ptr(), T)], _bb.ChecksumAlgo.BBH64, stream(), True)
        D = np.array(eng.debug_accumulators(), dtype=np.uint32).reshape(-1, 128, 16)[0]
        nz = np.argwhere(D.any(axis=1)).flatten()
        em, ek = _bb.bbh64_off_to_row(o), _bb.bbh64_off_to_k(o)
        expect = np.array([_bb.bbh64_weight(ek, n) for n in range(16)], dtype=np.uint32)
        good = len(nz) == 1 and nz[0] == em and np.array_equal(D[em], expect)
        ok_all &= good
        msg = f"impulse o={o:5d} expect(m={em:3d},k={ek:3d}) rows_nonzero={nz[:8].tolist()} "
        if len(nz) >= 1:
            row = D[nz[0]]
            # which k has this weight signature?
            cand = [k for k in range(128) if all(_bb.bbh64_weight(k, n) == int(row[n]) for n in range(16))]
            msg += f"hw_k={cand} vals={row[:4].tolist()}"
        print(("OK  " if good else "BAD ") + msg, "copy_ok", bool(torch.equal(src, dst)))
    print("IMPULSE_ALL_OK", ok_all)

    # ---- random objects
    sizes = [16, 48, 256, 4096, 5000, 16384, 16385, 16400, 100000, 1 << 20, (1 << 20) + 7, 3 * T + 33, 8 << 20]
    g = torch.Generator(device="cuda").manual_seed(1)
    all_ok = True
    for n in sizes:
        src = torch.randint(0, 256, (n + 64,), dtype=torch.uint8, device=dev, generator=g)[:n]
        dst = torch.full((n + 64,), 0xAB, dtype=torch.uint8, device=dev)
        dg, st, ms = eng.run([(src.data_ptr(), dst.data_ptr(), n)], _bb.ChecksumAlgo.BBH64, stream())
        torch.cuda.synchronize()
        ref = _bb.bbh64(src.cpu().numpy())
        copy_ok = bool(torch.equal(src, dst[:n])) and bool((dst[n:] == 0xAB).all())
        ok = (dg[0] == ref) and copy_ok and st[0] == 0
        all_ok &= ok
        print(("OK  " if ok else "BAD ") + f"n={n} digest={dg[0]:#x} ref={ref:#x} copy_ok={copy_ok} ms={ms:.3f}")
    print("RANDOM_ALL_OK", all_ok)
    all_ok = True
    for n in sizes + [64 << 20]:
        src = torch.randint(0, 256, (n + 64,), dtype=torch.uint8, device=dev, generator=g)[:n]
        dst = torch.full((n + 64,), 0xAB, dtype=torch.uint8, device=dev)
        dg, st, ms = eng.run([(src.data_ptr(), dst.data_ptr(), n)], _bb.ChecksumAlgo.CRC32C, stream())
        torch.cuda.synchronize()
        ref = _bb.crc32c(src.cpu().numpy())
        copy_ok = bool(torch.equal(src, dst[:n])) and bool((dst[n:] == 0xAB).all())
        dg2, st2, _ = eng.run([(src.data_ptr(), dst.data_ptr(), n, ref, _bb.XFER_VERIFY)], _bb.ChecksumAlgo.CRC32C, stream())
        dg3, st3, _ = eng.run([(src.data_ptr(), dst.data_ptr(), n, ref ^ 4, _bb.XFER_VERIFY)], _bb.ChecksumAlgo.CRC32C, stream())
        ok = (dg[0] == ref) and copy_ok and st2[0] == 0 and st3[0] == 1
        all_ok &= ok
        print(("OK  " if ok else "BAD ") + f"crc32c-fused n={n} digest={dg[0]:#x} ref={ref:#x} copy_ok={copy_ok} verify={st2[0]},{st3[0]} ms={ms:.3f}")
    print("CRC_FUSED_ALL_OK", all_ok)
    # an object large enough to straddle many CTAs (cross-CTA combine), both algos
    n = (300 << 20) + 12345
    src = torch.randint(0, 256, (n,), dtype=torch.uint8, device=dev, generator=g)
    dst = torch.empty(n, dtype=torch.uint8, device=dev)
    h = src.cpu().numpy()
    for algo, ref in ((_bb.ChecksumAlgo.BBH64, _bb.bbh64(h)), (_bb.ChecksumAlgo.CRC32C, _bb.crc32c(h))):
        dg, st, ms = eng.run([(src.data_ptr(), dst.data_ptr(), n)], algo, stream())
        print(("OK  " if dg[0] == ref else "BAD ") + f"straddle {algo.name} n={n} digest={dg[0]:#x} ref={ref:#x} copy_ok={bool(torch.equal(src, dst))} ms={ms:.3f} {n/ms/1e6:.0f} GB/s")
    del src, dst

    # ---- verify flag + 3 destinations + batch of small objects
    n = 123456 * 16
    src = torch.randint(0, 256, (n,), dtype=torch.uint8, device=dev, generator=g)
    d3 = [torch.zeros(n, dtype=torch.uint8, device=dev) for _ in range(3)]
    ref = _bb.bbh64(src.cpu().numpy())
    dg, st, ms = eng.run([(src.data_ptr(), [d.data_ptr() for d in d3], n, ref, _bb.XFER_VERIFY)], _bb.ChecksumAlgo.BBH64, stream())
    print("fanout3", dg[0] == ref, st[0], [bool(torch.equal(src, d)) for d in d3])
    dg, st, ms = eng.run([(src.data_ptr(), d3[0].data_ptr(), n, ref ^ 1, _bb.XFER_VERIFY)], _bb.ChecksumAlgo.BBH64, stream())
    print("verify_bad_expect -> status", st[0], "(want 1)")

    nobj, osz = 4096, 256
    big = torch.randint(0, 256, (nobj * osz,), dtype=torch.uint8, device=dev, generator=g)
    out = torch.zeros_like(big)
    items = [(big.data_ptr() + i * osz, out.data_ptr() + i * osz, osz) for i in range(nobj)]
    dg, st, ms = eng.run(items, _bb.ChecksumAlgo.BBH64, stream())
    h = big.cpu().numpy()
    bad = sum(1 for i in range(nobj) if dg[i] != _bb.bbh64(h[i * osz:(i + 1) * osz]))
    print(f"small-batch {nobj}x{osz}B bad_digests={bad} copy_ok={bool(torch.equal(big, out))} ms={ms:.3f}")
    # mixed sizes in one batch
    szs = [1 << 20, 256, 70000, 16, 16384, 33, 5 << 20, 4096]
    offs = np.cumsum([0] + [((s + 255) // 256) * 256 for s in szs])
    big = torch.randint(0, 256, (int(offs[-1]),), dtype=torch.uint8, device=dev, generator=g)
    out = torch.zeros_like(big)
    items = [(big.data_ptr() + int(offs[i]), out.data_ptr() + int(offs[i]), szs[i]) for i in range(len(szs))]
    dg, st, ms = eng.run(items, _bb.ChecksumAlgo.BBH64, stream())
    h = big.cpu().numpy()
    res = [dg[i] == _bb.bbh64(h[int(offs[i]):int(offs[i]) + szs[i]]) for i in range(len(szs))]
    cp = [bool(torch.equal(big[int(offs[i]):int(offs[i]) + szs[i]], out[int(offs[i]):int(offs[i]) + szs[i]])) for i in range(len(szs))]
    print("mixed-batch digests", res, "copies", cp)
    # copy-only algo
    out.zero_()
    dg, st, ms = eng.run(items, _bb.ChecksumAlgo.NONE, stream())
    cp = [bool(torch.equal(big[int(offs[i]):int(offs[i]) + szs[i]], out[int(offs[i]):int(offs[i]) + szs[i]])) for i in range(len(szs))]
    print("copy-only batch copies", cp)

    # ---- stand-alone CRC32C kernel
    for n in [1, 511, 512, 513, 4096, 100001, 1 << 22]:
        src = torch.randint(0, 256, (n,), dtype=torch.uint8, device=dev, generator=g)
        outc = torch.zeros(1, dtype=torch.int32, device=dev)
        scratch = torch.zeros((n + 511) // 512 + 1, dtype=torch.int32, device=dev)
        _bb.crc32c_device(src.data_ptr(), n, outc.data_ptr(), scratch.data_ptr(), stream())
        torch.cuda.synchronize()
        got = int(outc.item()) & 0xFFFFFFFF
        ref = _bb.crc32c(src.cpu().numpy())
        print(("OK  " if got == ref else "BAD ") + f"crc32c_device n={n} got={got:#x} ref={ref:#x}")


def timeit(fn, iters=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return min(ts), float(np.median(ts))


def phase_perf():
    dev = torch.device("cuda:0")
    eng = _bb.XferEngine(0, 1 << 16, 2)
    for nobj, osz in [(64, 16 << 20), (1024, 1 << 20), (16384, 65536), (65536, 4096), (65536, 256)]:
        total = nobj * osz
        src = torch.empty(total, dtype=torch.uint8, device=dev)
        _bb.random_fill(src.data_ptr(), total, 7, stream())
        dst = torch.empty(total, dtype=torch.uint8, device=dev)
        items = [(src.data_ptr() + i * osz, dst.data_ptr() + i * osz, osz) for i in range(nobj)]
        for algo in (_bb.ChecksumAlgo.BBH64, _bb.ChecksumAlgo.CRC32C, _bb.ChecksumAlgo.NONE):
            kms = []

            def run():
                dg, st, ms = eng.run(items, algo, stream())
                kms.append(ms)

            best, med = timeit(run)
            kbest = min(kms[2:])
            print(f"fused {algo.name:6s} {nobj:6d} x {osz:9d} B: kernel {kbest:8.3f} ms  {total / kbest / 1e6:8.1f} GB/s payload"
                  f" | end-to-end(submit+wait) {best:8.3f} ms {total / best / 1e6:8.1f} GB/s")
        if osz >= (1 << 20):
            best, med = timeit(lambda: _bb.copy_simt(dst.data_ptr(), src.data_ptr(), total, stream()))
            print(f"  simt copy (1 launch, whole buffer): {best:8.3f} ms {total / best / 1e6:8.1f} GB/s")
            best, med = timeit(lambda: dst.copy_(src))
            print(f"  torch copy_ (cudaMemcpy D2D)      : {best:8.3f} ms {total / best / 1e6:8.1f} GB/s")
            outc = torch.zeros(1, dtype=torch.int32, device=dev)
            scratch = torch.zeros(total // 512 + 2, dtype=torch.int32, device=dev)
            best, med = timeit(lambda: _bb.crc32c_device(src.data_ptr(), total, outc.data_ptr(), scratch.data_ptr(), stream()))
            print(f"  stand-alone crc32c kernel          : {best:8.3f} ms {total / best / 1e6:8.1f} GB/s")
        del src, dst
        torch.cuda.empty_cache()
    # CTA-count sensitivity on the big case
    nobj, osz = 64, 16 << 20
    total = nobj * osz
    src = torch.empty(total, dtype=torch.uint8, device=dev)
    _bb.random_fill(src.data_ptr(), total, 7, stream())
    dst = torch.empty(total, dtype=torch.uint8, device=dev)
    items = [(src.data_ptr() + i * osz, dst.data_ptr() + i * osz, osz) for i in range(nobj)]
    for ctas in (16, 32, 64, 96, 128, 132):
        eng.set_max_ctas(ctas)
        kms = []
        for _ in range(4):
            dg, st, ms = eng.run(items, _bb.ChecksumAlgo.BBH64, stream())
            kms.append(ms)
        print(f"ctas={ctas:4d}: {min(kms):8.3f} ms {total / min(kms) / 1e6:8.1f} GB/s")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("phase", choices=["probe", "perf"])
    a = ap.parse_args()
    t0 = time.time()
    print(torch.cuda.get_device_name(0), torch.version.cuda)
    try:
        {"probe": phase_probe, "perf": phase_perf}[a.phase]()
    except Exception:
        traceback.print_exc()
        sys.exit(1)
    print(f"phase {a.phase} done in {time.time() - t0:.1f}s")
