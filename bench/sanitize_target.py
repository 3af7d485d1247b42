#!/usr/bin/env python3
"""Small single-GPU target for compute-sanitizer (memcheck / synccheck / racecheck): every code path of the fused
transfer kernel on small inputs — three digest algorithms, verify, 3-way fan-out, odd sizes with byte tails, a
many-small-objects batch (table path) and single objects (inline-parameter path), plus the MXFP8 kernels."""
import sys

import torch

sys.path.insert(0, ".")
from blackbird_b200 import _bb  # noqa: E402

s = torch.cuda.current_stream().cuda_stream
eng = _bb.XferEngine(0, 4096, 2)
torch.manual_seed(0)
checked = 0
for algo, ref in ((_bb.ChecksumAlgo.XXH3, _bb.xxh3t64), (_bb.ChecksumAlgo.BBH64, _bb.bbh64), (_bb.ChecksumAlgo.CRC32C, _bb.crc32c), (_bb.ChecksumAlgo.NONE, None)):
    for n in (16, 255, 16384, 16400, 100_003, 1 << 20):
        cap = (n + 255) // 256 * 256
        src = torch.randint(0, 256, (cap,), dtype=torch.uint8, device="cuda")
        dsts = [torch.zeros(cap, dtype=torch.uint8, device="cuda") for _ in range(3)]
        dg, st, _ = eng.run([(src.data_ptr(), [d.data_ptr() for d in dsts], n)], algo, s)
        torch.cuda.synchronize()
        assert all(torch.equal(d[:n], src[:n]) for d in dsts)
        if ref is not None:
            assert dg[0] == ref(src[:n].cpu().numpy()), (algo, n)
            dg2, st2, _ = eng.run([(src.data_ptr(), dsts[0].data_ptr(), n, dg[0], _bb.XFER_VERIFY)], algo, s)
            assert st2 == [0]
        checked += 1
    # table path: 500 small objects of mixed sizes
    sizes = [(i * 37) % 3000 + 1 for i in range(500)]
    stride = 3072
    src = torch.randint(0, 256, (500 * stride,), dtype=torch.uint8, device="cuda")
    dst = torch.zeros_like(src)
    items = [(src.data_ptr() + i * stride, dst.data_ptr() + i * stride, sizes[i]) for i in range(500)]
    dg, st, _ = eng.run(items, algo, s)
    torch.cuda.synchronize()
    for i in (0, 1, 250, 499):
        assert torch.equal(src[i * stride:i * stride + sizes[i]], dst[i * stride:i * stride + sizes[i]])
        if ref is not None:
            assert dg[i] == ref(src[i * stride:i * stride + sizes[i]].cpu().numpy())
    checked += 1
    # the same objects padded past 4 KiB take the persistent kernel's table path; the ones above took the warp-per-object path
    sizes = [(i * 137) % 40000 + 1 for i in range(300)]
    stride = 40192
    src = torch.randint(0, 256, (300 * stride,), dtype=torch.uint8, device="cuda")
    d3 = [torch.zeros_like(src) for _ in range(3)]
    items = [(src.data_ptr() + i * stride, [d.data_ptr() + i * stride for d in d3[:1 + i % 3]], sizes[i]) for i in range(300)]
    dg, st, _ = eng.run(items, algo, s)
    torch.cuda.synchronize()
    for i in (0, 1, 2, 150, 299):
        for d in d3[:1 + i % 3]:
            assert torch.equal(src[i * stride:i * stride + sizes[i]], d[i * stride:i * stride + sizes[i]])
        if ref is not None:
            assert dg[i] == ref(src[i * stride:i * stride + sizes[i]].cpu().numpy())
    checked += 1
# resident mailbox warp: single small objects without a launch
eng.set_mailbox(True)
src = torch.randint(0, 256, (4096,), dtype=torch.uint8, device="cuda")
dst = torch.zeros_like(src)
for n in (1, 64, 1000, 4096):
    dg, st, _ = eng.run([(src.data_ptr(), dst.data_ptr(), n)], _bb.ChecksumAlgo.XXH3, s)
    assert dg[0] == _bb.xxh3t64(src[:n].cpu().numpy()) and torch.equal(src[:n], dst[:n])
eng.set_mailbox(False)
checked += 1
x = (torch.randn(4096 * 8, device="cuda") * 4).to(torch.bfloat16)
packed = torch.empty(_bb.mxfp8_packed_bytes(x.numel()), dtype=torch.uint8, device="cuda")
_bb.mxfp8_pack(x.data_ptr(), x.numel(), packed.data_ptr(), s)
back = torch.empty_like(x)
_bb.mxfp8_unpack(packed.data_ptr(), x.numel(), back.data_ptr(), s)
torch.cuda.synchronize()
assert (back.float() - x.float()).abs().max().item() <= x.float().abs().max().item() * 2 ** -3
# fused MXFP8 put gathering its elements from rows of 128 every 544 elements, starting 4 elements into row 0 (so every
# row segment has a head and a tail), into 2 replicas; compared with an unpatterned put of the compacted elements
flat = (torch.randn(64 * 544, device="cuda") * 4).to(torch.bfloat16)
n, row0 = 63 * 128, 132  # 2 * (row0 + 4) is 16-byte aligned
x = torch.arange(n, device="cuda") + 4
dense = flat[row0 + x // 128 * 544 + x % 128].contiguous()
reps = [torch.zeros(_bb.mxfp8_packed_bytes(n), dtype=torch.uint8, device="cuda") for _ in range(3)]
dg, st, _ = eng.run_fp8([(flat.data_ptr() + 2 * row0, [r.data_ptr() for r in reps[:2]], n, None, None, (544, 128, 4))], False, s)
dg2, _, _ = eng.run_fp8([(dense.data_ptr(), reps[2].data_ptr(), n)], False, s)
torch.cuda.synchronize()
assert dg == dg2 and torch.equal(reps[0], reps[2]) and torch.equal(reps[1], reps[2])
# scattering store of bb_xfer: an object stored into rows of 100 every 132 bytes, starting 4 bytes into row 0 (so every row
# segment has a head and a tail), verified; the gaps keep their guard
n = 3 * 16384 + 77
src = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda")
gdst = torch.full(((n + 4) // 100 * 132 + 256,), 0xA5, dtype=torch.uint8, device="cuda")
x = torch.arange(n, device="cuda") + 4
at = 12 + x // 100 * 132 + x % 100  # row 0 at byte 12 of gdst, so that row 0 + phase is 16-byte aligned
dg, st, _ = eng.run([(src.data_ptr(), gdst.data_ptr() + 12, n, _bb.xxh3t64(src.cpu().numpy()), _bb.XFER_VERIFY, 0, None, None,
                      (132, 100, 4))], _bb.ChecksumAlgo.XXH3, s)
torch.cuda.synchronize()
mask = torch.ones_like(gdst, dtype=torch.bool)
mask[at] = False
assert st == [0] and torch.equal(gdst[at], src) and bool((gdst[mask] == 0xA5).all())
# scattering store of the fused MXFP8 unpack: the packed object above unpacked into rows of 128 every 544 elements from
# element 4 of row 0, compared with a plain unpack scattered by torch
out = torch.full((64 * 544,), -7.0, dtype=torch.bfloat16, device="cuda")
plain = torch.empty(63 * 128, dtype=torch.bfloat16, device="cuda")
eng.run_fp8([(plain.data_ptr(), reps[2].data_ptr(), 63 * 128)], True, s)
dg3, st3, _ = eng.run_fp8([(out.data_ptr() + 2 * row0, reps[2].data_ptr(), 63 * 128, dg2[0], None, None, (544, 128, 4))], True, s)
torch.cuda.synchronize()
x = torch.arange(63 * 128, device="cuda") + 4
at = row0 + x // 128 * 544 + x % 128
mask = torch.ones_like(out, dtype=torch.bool)
mask[at] = False
assert st3 == [0] and torch.equal(out[at].view(torch.int16), plain.view(torch.int16)) and bool((out[mask] == -7.0).all())
print(f"sanitize target OK: {checked} kernel configurations + mxfp8 + gathered mxfp8 put + scattered get + scattered mxfp8 get")
