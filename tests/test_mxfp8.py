"""MXFP8 (E4M3 + E8M0/32) CPU reference vs an independent torch model; GPU kernels vs the CPU reference."""
import numpy as np
import pytest
import torch


def test_e4m3_conversion_matches_torch_float8(bb):
    vals = torch.cat([torch.linspace(-500, 500, 4001), torch.tensor([0.0, 1e-9, 2 ** -9, 2 ** -10, 1.5 * 2 ** -9, 2 ** -6, 447.9, 448.0, 464.0, 1e6]),
                      torch.randn(5000) * 3, torch.randn(2000) * 0.01])
    ref = vals.clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
    got = torch.tensor([bb.e4m3_from_float(float(v)) for v in vals], dtype=torch.uint8)
    # -0.0 vs +0.0 encodings may differ for tiny negatives that round to zero
    same = (got == ref) | (((got & 0x7F) == 0) & ((ref & 0x7F) == 0))
    assert bool(same.all()), vals[~same][:10]
    for b in range(256):
        if (b & 0x7F) == 0x7F:
            continue
        assert bb.e4m3_to_float(b) == float(torch.tensor([b], dtype=torch.uint8).view(torch.float8_e4m3fn).float())


def _torch_mx_reference(x_bf16: torch.Tensor):
    x = x_bf16.float().view(-1, 32)
    amax = x.abs().amax(dim=1)
    exp = torch.where(amax > 0, torch.floor(torch.log2(amax)) - 8, torch.zeros_like(amax))
    scale = torch.exp2(exp)
    q = (x / scale[:, None]).clamp(-448, 448).to(torch.float8_e4m3fn)
    return q.view(torch.uint8).view(-1), (exp + 127).clamp(0, 254).to(torch.uint8), (q.float() * scale[:, None]).view(-1)


def test_pack_reference_matches_torch_model(bb):
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(32 * 512, generator=g) * torch.logspace(-4, 3, 32 * 512)).to(torch.bfloat16)
    x[:32] = 0  # all-zero block
    packed = np.frombuffer(bb.mxfp8_pack_ref(x.view(torch.int16).numpy()), dtype=np.uint8)
    n = x.numel()
    assert len(packed) == bb.mxfp8_packed_bytes(n) == n + n // 32
    q_ref, s_ref, deq_ref = _torch_mx_reference(x)
    assert np.array_equal(packed[n:], s_ref.numpy())
    pay = torch.from_numpy(packed[:n].copy())
    same = (pay == q_ref) | (((pay & 0x7F) == 0) & ((q_ref & 0x7F) == 0))
    assert bool(same.all())
    back = torch.frombuffer(bytearray(bb.mxfp8_unpack_ref(packed, n)), dtype=torch.bfloat16).float()
    assert torch.allclose(back, deq_ref.to(torch.bfloat16).float(), rtol=0, atol=0)
    # quantisation error bound: E4M3 has 3 mantissa bits -> relative error <= 2^-4 of the block max scale
    err = (back - x.float()).abs().view(-1, 32).amax(dim=1)
    bound = x.float().abs().view(-1, 32).amax(dim=1) * 2 ** -3 + 1e-30
    assert bool((err <= bound).all())


# Blocks with special values (bf16 bit patterns): +-Inf, NaN of either sign, subnormals, negative zeros, and mixes of them
# with normal values; the block maximum skips NaN, an Inf selects the neutral scale.
SPECIAL_BLOCKS = np.array([
    [0x7F80, 0x3F80, 0xC000] + [0x3E00] * 29,    # +Inf with normals
    [0xFF80, 0x4100, 0x0001] + [0xBC00] * 29,    # -Inf with a normal and a subnormal
    [0x7FC0, 0x4000, 0xC040] + [0x3C00] * 29,    # NaN with normals
    [0xFFC1, 0x7FC0] + [0xFFC0] * 30,            # NaN only
    [0x0001, 0x8003, 0x007F, 0x8040] * 8,        # subnormals only (the scale clamps at 0)
    [0x0001, 0x807F, 0x3F80, 0x8000] * 8,        # subnormals and -0 next to 1.0
    [0x8000] * 32,                               # negative zeros only
    [0x8000, 0x0000, 0x0080, 0x8080] * 8,        # +-0 and +-the smallest normal (the scale clamps at 0)
], dtype=np.uint16)


def special_blocks(rows=slice(None)):
    """SPECIAL_BLOCKS[rows] as one flat bf16 tensor on the GPU."""
    return torch.from_numpy(SPECIAL_BLOCKS[rows].reshape(-1).view(np.int16).copy()).view(torch.bfloat16).cuda()


def check_packed(got, ref, n, what=""):
    """Stored MXFP8 object (numpy uint8) vs mxfp8_pack_ref: block scales and payload identical, the sign of a zero
    included (a negative element that rounds to zero is stored as -0, 0x80)."""
    assert np.array_equal(got[n:], ref[n:]), f"{what}: block scales differ at {np.nonzero(got[n:] != ref[n:])[0][:10]}"
    diff = got[:n] != ref[:n]
    assert not diff.any(), f"{what}: payload differs at {np.nonzero(diff)[0][:10]}"


def check_unpacked(bb, back, packed, n, what=""):
    """Dequantised bf16 (CPU tensor) vs mxfp8_unpack_ref of the same packed bytes: bit for bit, every block scale included;
    NaN is compared only as NaN (the NaN bit patterns of the two sides differ)."""
    ref = torch.frombuffer(bytearray(bb.mxfp8_unpack_ref(packed, n)), dtype=torch.bfloat16)
    nan = ref.isnan()
    assert torch.equal(back.isnan(), nan), f"{what}: NaN positions differ"
    bad = back.view(torch.int16) != ref.view(torch.int16)
    bad &= ~nan
    assert not bool(bad.any()), f"{what}: elements {bad.nonzero().flatten()[:10].tolist()} differ"


@pytest.mark.gpu
def test_gpu_pack_unpack_match_cpu_reference_at_every_block_scale(bb):
    """mxfp8_pack / mxfp8_unpack against the CPU reference: stored bytes, and dequantised values bit for bit at every block
    scale, 0 (2^-127, an fp32 subnormal) included."""
    assert torch.cuda.is_available()
    g = torch.Generator(device="cuda").manual_seed(1)
    n = 32 * 40000 + 32 * 3
    x = (torch.randn(n, device="cuda", generator=g) * 10 ** torch.empty(n, device="cuda").uniform_(-3, 2, generator=g)).to(torch.bfloat16)
    x[64:96] = 0
    nx, x = n, torch.cat([x, special_blocks()])
    n = x.numel()
    packed = torch.zeros(bb.mxfp8_packed_bytes(n), dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    bb.mxfp8_pack(x.data_ptr(), n, packed.data_ptr(), s)
    torch.cuda.synchronize()
    ref = np.frombuffer(bb.mxfp8_pack_ref(x.cpu().view(torch.int16).numpy()), dtype=np.uint8)
    got = packed.cpu().numpy()
    check_packed(got, ref, n)
    out = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
    bb.mxfp8_unpack(packed.data_ptr(), n, out.data_ptr(), s)
    torch.cuda.synchronize()
    assert bool((got[n:] == 0).any())  # blocks whose scale is 0 (2^-127) are among those compared
    check_unpacked(bb, out.cpu(), got, n)
    # fp32 reference of the op: dequantised values stay within the E4M3 error bound
    err = (out[:nx].float() - x[:nx].float()).abs().view(-1, 32).amax(dim=1)
    assert bool((err <= x[:nx].float().abs().view(-1, 32).amax(dim=1) * 2 ** -3 + 1e-30).all())


@pytest.mark.gpu
def test_fused_fp8_put_get_matches_unfused_pack_and_cpu_digest(bb):
    """bb_xfer_fp8: pack fused into the put (bf16 read once, E4M3 payload hashed on the tensor cores in shared memory)
    and unpack fused into the get.  The stored bytes and the digest must be identical to mxfp8_pack + bbh64."""
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need CUDA (marked gpu)")
    s = torch.cuda.current_stream().cuda_stream
    eng = bb.XferEngine(0, 1024, 2)
    torch.manual_seed(3)
    sizes = [16384, 16384 * 5, 16384 * 64 + 16384 * 3]
    xs = [(torch.randn(n, device="cuda") * (1 + i)).to(torch.bfloat16) for i, n in enumerate(sizes)]
    xs[1][100:132] = 0  # an all-zero block
    xs[2][7] = float("inf")
    slabs = [torch.zeros(bb.mxfp8_packed_bytes(n), dtype=torch.uint8, device="cuda") for n in sizes]
    assert all(bb.XferEngine.fp8_eligible(n) for n in sizes) and bb.XferEngine.fp8_eligible(16384 + 32) and not bb.XferEngine.fp8_eligible(16384 + 8)
    dg, st, ms = eng.run_fp8([(x.data_ptr(), sl.data_ptr(), n) for x, sl, n in zip(xs, slabs, sizes)], False, s)
    torch.cuda.synchronize()
    for x, sl, n, d in zip(xs, slabs, sizes, dg):
        ref = torch.empty_like(sl)
        bb.mxfp8_pack(x.data_ptr(), n, ref.data_ptr(), s)
        torch.cuda.synchronize()
        assert torch.equal(sl, ref), n  # byte-identical to the stand-alone pack kernel
        assert d == bb.bbh64(sl.cpu().numpy()), n  # digest of the stored packed object
    outs = [torch.zeros_like(x) for x in xs]
    dg2, st2, _ = eng.run_fp8([(o.data_ptr(), sl.data_ptr(), n, d) for o, sl, n, d in zip(outs, slabs, sizes, dg)], True, s)
    torch.cuda.synchronize()
    assert st2 == [0, 0, 0] and dg2 == dg
    for x, sl, n, o in zip(xs, slabs, sizes, outs):
        ref = torch.empty_like(x)
        bb.mxfp8_unpack(sl.data_ptr(), n, ref.data_ptr(), s)
        torch.cuda.synchronize()
        assert torch.equal(o.view(torch.int16), ref.view(torch.int16)), n
    slabs[1][5000] ^= 0x40  # corrupt the payload, and the scales of another object
    slabs[2][sizes[2] + 17] ^= 0x01
    _, st3, _ = eng.run_fp8([(o.data_ptr(), sl.data_ptr(), n, d) for o, sl, n, d in zip(outs, slabs, sizes, dg)], True, s)
    assert st3 == [0, 1, 1]


@pytest.mark.gpu
def test_standalone_kernels_at_their_grid_stride_edges(bb):
    """mxfp8_pack / mxfp8_unpack are grid-stride loops over 16-byte chunks (4 per block) on at most 8 CTAs of 256 threads
    per SM, and the pack pads its trip count to whole warps.  Objects of one to four blocks (a partial warp), and chunk
    counts one block below, at and one block above what one pass of the largest grid covers, each ending in special-value
    blocks: stored bytes, dequantised values and the bytes past both outputs against the CPU reference."""
    assert torch.cuda.is_available()
    s = torch.cuda.current_stream().cuda_stream
    one_pass = torch.cuda.get_device_properties(0).multi_processor_count * 8 * 256  # chunks covered by the largest grid
    g = torch.Generator(device="cuda").manual_seed(11)
    for i, n in enumerate([32, 64, 96, 128] + [8 * (one_pass + d) for d in (-4, 0, 4)]):
        x = (torch.randn(n, device="cuda", generator=g) * 10 ** torch.empty(n, device="cuda").uniform_(-4, 3, generator=g)).to(torch.bfloat16)
        sp = special_blocks([(k + 3 * i) % 8 for k in range(min(n // 32, 8))])
        x[n - sp.numel():] = sp
        m = bb.mxfp8_packed_bytes(n)
        packed = torch.full((m + 64,), 0xA5, dtype=torch.uint8, device="cuda")
        out = torch.full((n + 32,), 0x5A5A, dtype=torch.int16, device="cuda")
        bb.mxfp8_pack(x.data_ptr(), n, packed.data_ptr(), s)
        bb.mxfp8_unpack(packed.data_ptr(), n, out.data_ptr(), s)
        torch.cuda.synchronize()
        got = packed.cpu().numpy()
        check_packed(got[:m], np.frombuffer(bb.mxfp8_pack_ref(x.cpu().view(torch.int16).numpy()), dtype=np.uint8), n, f"n={n}")
        assert bool((got[m:] == 0xA5).all()), f"n={n}: the pack wrote past the packed object"
        back = out.cpu()
        check_unpacked(bb, back[:n].view(torch.bfloat16), got[:m], n, f"n={n}")
        assert bool((back[n:] == 0x5A5A).all()), f"n={n}: the unpack wrote past the output"
