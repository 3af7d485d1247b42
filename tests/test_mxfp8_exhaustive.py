"""MXFP8 pack and unpack, exhaustively, against an exact model of the format, through every implementation that encodes or
decodes it: the CPU reference (common/mxfp8.cpp), the stand-alone kernels (mxfp8.cu), the fused pack with 1-3 replicas,
the fused gathered pack, the fused unpack (whole object, element window, strided window) and TensorStore.

The model below is written from the rule in common/mxfp8.h, in float64 numpy on bf16 bit patterns.  Every product it
forms is a power of two times at most 8 significant bits, so float64 holds it exactly and the only roundings are the
ones the format defines: RNE onto the E4M3 grid (saturating at +-448) and RNE onto the bf16 grid.  It is checked
against torch's float8_e4m3fn and bfloat16 conversions, a third implementation, on every value it is used on.

Three input sets reach the whole format:
  P  every finite bf16 x under the block scale of every bf16 binade b with |x| <= amax(b): all 255 exponent fields, so
     block scales 0..246 (the largest a finite bf16 gives), with the block maximum rotated through every lane position;
  S  blocks of special values (NaN of either sign and payload, +-Inf, +-0, subnormals) around a maximum at each of the
     32 positions of a block;
  U  every (E4M3 byte, E8M0 byte) pair: 256 scales x 256 payload bytes, in 4 whole tiles, and again rotated with a
     tail tile that holds a block of every scale.
Every kernel result must equal the model bit for bit: scale bytes, payload bytes with the sign of zero, and dequantised
bf16 patterns; a NaN is compared as a NaN only."""
import numpy as np
import pytest
import torch

T = 16384  # elements per payload tile of the fused kernels
GAP_FILL = np.array([0x7FC0, 0xFF80, 0x7F7F, 0x7F80, 0xFFC1, 0xFF7F], dtype=np.uint16)  # NaN, +-Inf, +-bf16 max


# ---------------------------------------------------------------------------------------------------- the model


def bf16_value(bits):
    """float64 value of bf16 bit patterns (exact)."""
    with np.errstate(invalid="ignore"):  # signalling NaN patterns
        return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def model_scales(x):
    """E8M0 byte of every 32-element block of bf16 patterns x: clamp(floor(log2 amax) - 8 + 127, 0, 254), amax over the
    block skipping NaN; 127 for a block whose amax is 0 (all zeros or all NaN) or Inf.  floor(log2 amax) comes from the
    exponent field, so a subnormal amax (field 0) clamps to 0."""
    mag = (x.reshape(-1, 32) & 0x7FFF).astype(np.int32)
    amax = np.where(mag > 0x7F80, -1, mag).max(axis=1)
    e = np.clip((amax >> 7) - 127 - 8 + 127, 0, 254)
    return np.where((amax <= 0) | (amax == 0x7F80), 127, e).astype(np.uint8)


def model_scaled(x):
    """(scale bytes, x * 2^(127 - scale) per element as float64): the exact values the E4M3 encoding rounds."""
    s = model_scales(x)
    return s, (bf16_value(x).reshape(-1, 32) * np.ldexp(1.0, 127 - s.astype(np.int64))[:, None]).reshape(-1)


def e4m3_encode(v):
    """E4M3 bytes of float64 values: RNE onto the grid of step 2^(max(floor(log2|v|), -6) - 3), saturated to +-448;
    NaN -> 0x7F, +-Inf -> 0x7E / 0xFE, and a negative value that rounds to zero -> 0x80 (-0)."""
    nan = np.isnan(v)
    a = np.where(nan, 0.0, np.abs(v))
    _, ex = np.frexp(a)  # a = m * 2^ex, m in [0.5, 1): floor(log2 a) = ex - 1
    step = np.ldexp(1.0, np.maximum(ex - 1, -6) - 3)
    q = np.minimum(np.rint(a / step) * step, 448.0)
    _, qe = np.frexp(q)
    normal = q >= 2.0 ** -6
    man = np.where(normal, q * np.ldexp(1.0, 1 - qe) * 8 - 8, q * 512).astype(np.int64)
    code = (np.where(normal, qe - 1 + 7, 0).astype(np.int64) << 3) | man | (np.signbit(v).astype(np.int64) << 7)
    return np.where(nan, 0x7F, code).astype(np.uint8)


def e4m3_decode(b):
    """float64 value of E4M3 bytes (0x7F / 0xFF are NaN)."""
    b = np.asarray(b, dtype=np.uint8).astype(np.int64)
    e, m = (b >> 3) & 15, b & 7
    mag = np.where(e == 0, m * 2.0 ** -9, np.ldexp(1.0 + m / 8.0, e - 7))
    return np.where((b & 0x7F) == 0x7F, np.nan, np.where(b & 0x80, -mag, mag))


def bf16_encode(w):
    """bf16 patterns of float64 values: RNE onto the grid of step 2^(max(floor(log2|w|), -126) - 7) (subnormal step
    2^-133); values at or past (2 - 2^-8) * 2^127 become +-Inf; NaN -> 0x7FC0."""
    nan = np.isnan(w)
    a = np.where(nan, 0.0, np.abs(w))
    _, ex = np.frexp(np.where(np.isinf(a), 0.0, a))
    step = np.ldexp(1.0, np.maximum(ex - 1, -126) - 7)
    q = np.rint(a / step) * step
    q = np.copysign(np.where(q >= 2.0 ** 128, np.inf, q), w)
    bits = (np.where(nan, 0.0, q).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
    return np.where(nan, np.uint16(0x7FC0), bits)


def model_pack(x):
    """[E4M3 payload n | E8M0 scales n/32] of bf16 patterns x (n a multiple of 32)."""
    s, v = model_scaled(x)
    return np.concatenate([e4m3_encode(v), s])


def model_products(packed, n):
    """decode(byte) * 2^(scale - 127) per element, exact.  Scale byte 255 is never packed; the implementations read it
    as 2^128, which overflows fp32, so the model gives them +-Inf, and NaN for a zero payload (0 * Inf)."""
    s = packed[n:n + n // 32].astype(np.int64)
    f = np.where(s == 255, np.inf, np.ldexp(1.0, np.minimum(s, 254) - 127))
    with np.errstate(invalid="ignore"):
        return (e4m3_decode(packed[:n]).reshape(-1, 32) * f[:, None]).reshape(-1)


def model_unpack(packed, n):
    """Dequantised bf16 patterns of a packed object."""
    return bf16_encode(model_products(packed, n))


def same_bits(got, want, kind, what):
    """Fails unless got equals want bit for bit: kind "e4m3" (payload bytes), "bf16" (uint16 / int16 patterns) or
    "e8m0" (scale bytes).  The sign of zero counts; a NaN only has to be a NaN (implementations encode it differently)."""
    got, want = np.asarray(got).reshape(-1), np.asarray(want).reshape(-1)
    assert got.shape == want.shape, f"{what}: {got.shape} elements, want {want.shape}"
    if kind == "bf16":
        got, want = got.view(np.uint16), want.view(np.uint16)
        gnan, wnan = (got & 0x7FFF) > 0x7F80, (want & 0x7FFF) > 0x7F80
    elif kind == "e4m3":
        gnan, wnan = (got & 0x7F) == 0x7F, (want & 0x7F) == 0x7F
    else:
        gnan = wnan = np.zeros(got.shape, dtype=bool)
    bad = (gnan != wnan) | (~wnan & (got != want))
    if bad.any():
        i = np.nonzero(bad)[0][:8]
        pytest.fail(f"{what}: {int(bad.sum())} of {bad.size} {kind} values differ, at {i.tolist()}: "
                    f"got {[hex(v) for v in got[i]]}, want {[hex(v) for v in want[i]]}")


def check_packed(got, want, n, what):
    """A packed object against the model's: scale bytes exactly, then the payload (NaN as NaN)."""
    same_bits(got[n:], want[n:], "e8m0", f"{what}: block scales")
    same_bits(got[:n], want[:n], "e4m3", f"{what}: payload")


# ---------------------------------------------------------------------------------------------------- the input sets


def pack_sweep():
    """P: for every exponent field b in 0..254, every finite bf16 x with |x| <= top(b) = the largest bf16 with field b, in
    blocks of 31 next to an anchor that is the block maximum.  Blocks take the anchor top(b), or exactly 2^(b - 127)
    (the smallest subnormal for b = 0) when all their elements are at most that.  Block j puts its anchor at position
    j % 32 with sign (-1)^(j // 32), so the maximum sits in every lane and half-word of pack_chunk's 4-lane shuffle."""
    rng = np.random.default_rng(0)
    fills, anchors = [], []
    for b in range(255):
        top, low = (b << 7) | 0x7F, (b << 7) if b else 0x0001
        mags = np.arange(top + 1, dtype=np.uint16)
        xs = np.concatenate([mags, mags | 0x8000])
        rng.shuffle(xs)
        under = (xs & 0x7FFF) <= low
        k = int(under.sum()) // 2  # half of the elements at most 2^k go with that anchor
        lo_set = xs[under][:k]
        hi_set = xs[~(under & (np.cumsum(under) <= k))]
        for group, anchor in ((hi_set, top), (lo_set, low)):
            if group.size == 0:
                continue
            nb = -(-group.size // 31)
            fills.append(np.resize(group, nb * 31).reshape(nb, 31))  # the last block is topped up from the group's start
            anchors.append(np.full(nb, anchor, dtype=np.uint16))
    fill, anchor = np.concatenate(fills), np.concatenate(anchors)
    j = np.arange(anchor.size)
    anchor |= ((j >> 5) & 1).astype(np.uint16) << 15
    at = np.arange(32)[None, :] == (j % 32)[:, None]
    out = np.empty((anchor.size, 32), dtype=np.uint16)
    out[at] = anchor
    out[~at] = fill.reshape(-1)
    return out.reshape(-1)


def special_sweep():
    """S: for every position p of a block, blocks whose distinguished element at p is a positive maximum, a negative
    maximum, a negative maximum with its positive twin elsewhere, +Inf, -Inf, or a NaN (0x7FC0, 0xFFC1, 0x7F81, whose
    magnitude above 0x7F80 must be skipped, not taken as the maximum); the other 31 elements mix NaN, +-0, subnormals
    and normals below the maximum.  Then blocks that are all NaN, all +-0, or subnormals only, each with its extreme at
    p."""
    rows = []
    for p in range(32):
        m = ((40 + 6 * p) << 7) | (p * 5 % 128)  # the maximum's magnitude: exponent fields 40..226
        fill = np.array([0x0000, 0x8000, 0x0001, 0x8001, 0x007F, 0x807F, 0x0080, 0x8080, 0x7FC0, 0xFFC1, 0x7F81, 0xFFFF]
                        + [(m - k * 0x93) | (0x8000 if k % 2 else 0) for k in range(1, 20)], dtype=np.uint16)
        fill = np.roll(fill, 5 * p)

        def block(v, others=fill):
            return np.insert(others, p, v)

        twin = block(m | 0x8000)
        twin[(p + 13) % 32] = m
        rows += [block(m), block(m | 0x8000), twin, block(0x7F80), block(0xFF80), block(0x7FC0), block(0xFFC1), block(0x7F81),
                 block(0x7F81, np.resize(np.array([0x7FC0, 0xFFC1, 0xFFFF, 0x7FFF, 0xFF81], dtype=np.uint16), 31)),
                 block(0x8000, np.resize(np.array([0x0000, 0x8000], dtype=np.uint16), 31)),
                 block(0x807F, (np.arange(1, 32, dtype=np.uint16) * 4) | np.where(np.arange(31) % 2, 0x8000, 0).astype(np.uint16))]
    return np.concatenate(rows)


def unpack_tables():
    """U: packed objects holding every (payload byte, scale byte) pair.  The first has 2048 blocks (4 whole tiles), block
    s * 8 + g with scale s and payload bytes 32g..32g+31.  The second is the first rotated by 777 blocks, then 263
    more: one block of every scale, and 7 of scales 0, 1, 126, 127, 128, 246 and 255, so that every scale also lands in
    a tail tile, whose last scale bytes are no 16-byte multiple.  Returns [(packed, n)]."""
    payload = np.tile(np.arange(256, dtype=np.uint8), 256).reshape(-1, 32)
    scales = np.repeat(np.arange(256, dtype=np.uint8), 8)
    extra_s = np.concatenate([np.arange(256), [0, 1, 126, 127, 128, 246, 255]]).astype(np.uint8)
    extra_g = np.concatenate([(np.arange(256) * 3 + 1) % 8, np.arange(7)])
    extra_p = (extra_g[:, None] * 32 + np.arange(32)[None, :]).astype(np.uint8)
    p2 = np.concatenate([np.roll(payload, 777, axis=0), extra_p])
    s2 = np.concatenate([np.roll(scales, 777), extra_s])
    return [(np.concatenate([payload.reshape(-1), scales]), payload.size), (np.concatenate([p2.reshape(-1), s2]), p2.size)]


@pytest.fixture(scope="module")
def sweeps():
    """The input sets and the model's results on them, built once per module."""
    P, S, U = pack_sweep(), special_sweep(), unpack_tables()
    P_packed, S_packed = model_pack(P), model_pack(S)
    return {"P": P, "S": S, "U": U, "P_packed": P_packed, "S_packed": S_packed,
            "P_back": model_unpack(P_packed, P.size), "U_back": [model_unpack(u, n) for u, n in U]}


# ---------------------------------------------------------------------------------------------------- CPU


def test_sweeps_cover_every_scale_and_every_pair(sweeps):
    """P reaches every scale byte a finite bf16 can produce, and every block of P has its anchor as its maximum; U holds
    all 65,536 (payload, scale) pairs, and its second object's tail tile a block of every scale."""
    P, n = sweeps["P"], sweeps["P"].size
    assert n % 32 == 0 and 8_000_000 < n < 9_000_000
    assert np.array_equal(np.unique(sweeps["P_packed"][n:]), np.arange(247))
    assert (P.reshape(-1, 32) & 0x7FFF).max() == 0x7F7F and not ((P & 0x7FFF) >= 0x7F80).any()  # P is finite
    pos = np.argmax(P.reshape(-1, 32) & 0x7FFF, axis=1)  # the first position holding the block maximum
    assert np.array_equal(np.unique(pos), np.arange(32))
    for u, m in sweeps["U"]:
        pairs = u[:m].astype(np.int64) * 256 + np.repeat(u[m:], 32)
        assert np.unique(pairs).size == 65536
    u, m = sweeps["U"][1]
    tail = 4 * T
    assert m > tail and np.array_equal(np.unique(u[m + tail // 32:]), np.arange(256)) and (m - tail) // 32 % 16 != 0


def test_model_matches_torch_float8_and_bfloat16(sweeps):
    """The model's E4M3 encoding of the scaled elements of P and S equals torch's float8_e4m3fn (after a clamp to +-448),
    and its bf16 rounding of the dequantised products of P's packing and of U equals torch's bfloat16 conversion."""
    for name in ("P", "S"):
        _, v = model_scaled(sweeps[name])
        ref = torch.from_numpy(v).clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8).numpy()
        same_bits(e4m3_encode(v), ref, "e4m3", f"{name}: E4M3 vs torch")
    n = sweeps["P"].size
    objs = [(sweeps["P_packed"], n)] + sweeps["U"]
    for i, (packed, m) in enumerate(objs):
        w = model_products(packed, m)
        ref = torch.from_numpy(w).to(torch.bfloat16).view(torch.int16).numpy()
        same_bits(bf16_encode(w), ref, "bf16", f"object {i}: bf16 vs torch")


def test_cpu_reference_matches_model(bb, sweeps):
    """mxfp8_pack_ref on P and S, mxfp8_unpack_ref on U and on the model's packing of P, and e4m3_from_float on every
    distinct scaled element of P and S."""
    for name in ("P", "S"):
        x = sweeps[name]
        check_packed(np.frombuffer(bb.mxfp8_pack_ref(x), dtype=np.uint8), sweeps[f"{name}_packed"], x.size, f"mxfp8_pack_ref({name})")
        _, v = model_scaled(x)
        v = np.unique(v.view(np.uint64)).view(np.float64)  # by bit pattern: -0 and +0 both stay
        got = np.array([bb.e4m3_from_float(float(f)) for f in v], dtype=np.uint8)
        same_bits(got, e4m3_encode(v), "e4m3", f"e4m3_from_float on the scaled elements of {name}")
    n = sweeps["P"].size
    got = np.frombuffer(bb.mxfp8_unpack_ref(sweeps["P_packed"], n), dtype=np.uint16)
    same_bits(got, sweeps["P_back"], "bf16", "mxfp8_unpack_ref(model packing of P)")
    for i, ((u, m), back) in enumerate(zip(sweeps["U"], sweeps["U_back"])):
        same_bits(np.frombuffer(bb.mxfp8_unpack_ref(u, m), dtype=np.uint16), back, "bf16", f"mxfp8_unpack_ref(U{i})")


# ---------------------------------------------------------------------------------------------------- GPU


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _dev(a):
    """A numpy array on the GPU (same bytes)."""
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()


def _host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need CUDA (marked gpu)")


@pytest.fixture(scope="module")
def _engine(cuda):
    from blackbird_b200 import _bb

    return _bb.XferEngine(0, 4096, 2)


@pytest.mark.gpu
def test_standalone_pack_matches_model(bb, sweeps, cuda):
    """mxfp8_pack on P and S."""
    for name in ("P", "S"):
        x = sweeps[name]
        n = x.size
        out = torch.empty(bb.mxfp8_packed_bytes(n), dtype=torch.uint8, device="cuda")
        bb.mxfp8_pack(_dev(x).data_ptr(), n, out.data_ptr(), _stream())
        check_packed(_host(out), sweeps[f"{name}_packed"], n, f"mxfp8_pack({name})")


@pytest.mark.gpu
def test_standalone_unpack_matches_model(bb, sweeps, cuda):
    """mxfp8_unpack on U and on the model's packing of P."""
    objs = [(sweeps["P_packed"], sweeps["P"].size, sweeps["P_back"])] + [u + (b,) for u, b in zip(sweeps["U"], sweeps["U_back"])]
    for i, (packed, n, back) in enumerate(objs):
        out = torch.empty(n, dtype=torch.int16, device="cuda")
        bb.mxfp8_unpack(_dev(packed).data_ptr(), n, out.data_ptr(), _stream())
        same_bits(_host(out), back, "bf16", f"mxfp8_unpack(object {i})")


@pytest.mark.gpu
def test_fused_pack_matches_model(bb, sweeps, _engine):
    """The fused pack (bb_xfer_fp8 put) of P and S into 3 replicas: every replica holds the model's packing, and the
    digest is bbh64 of the model's packed bytes, a packing made without any kernel."""
    xs = [sweeps["P"], sweeps["S"]]
    want = [sweeps["P_packed"], sweeps["S_packed"]]
    srcs = [_dev(x) for x in xs]
    reps = [[torch.full((w.size,), 0xA5, dtype=torch.uint8, device="cuda") for _ in range(3)] for w in want]
    dg, st, _ = _engine.run_fp8([(s.data_ptr(), [r.data_ptr() for r in rs], x.size) for s, rs, x in zip(srcs, reps, xs)], False, _stream())
    assert st == [0, 0]
    for name, x, w, rs, d in zip("PS", xs, want, reps, dg):
        got = [_host(r) for r in rs]
        assert all(np.array_equal(g, got[0]) for g in got[1:]), f"{name}: the replicas differ"
        check_packed(got[0], w, x.size, f"fused pack({name})")
        assert d == bb.bbh64(w), f"{name}: digest"


def gathered_source(x, pitch, width, phase):
    """(device buffer, pointer offset in elements) holding x as rows of `width` elements every `pitch` elements, the
    pattern's row 0 starting `phase` elements before x[0] (at a 16-byte aligned address); every element outside the rows
    cycles through NaN, +-Inf and +-bf16 max, so a gap element read by mistake changes its block's scale or payload."""
    y = np.arange(x.size, dtype=np.int64) + phase
    idx = y // width * pitch + y % width
    off = (8 - phase % 8) % 8
    buf = np.resize(GAP_FILL, off + int(idx[-1]) + 1 + 64)
    buf[off + idx] = x
    return _dev(buf), off


@pytest.mark.gpu
def test_fused_gathered_pack_matches_model(bb, sweeps, _engine):
    """The fused pack reading P from rows of 8 and of 40 elements (XFER_GATHER), the gaps between rows full of NaN, Inf
    and bf16 max: the packed bytes and the digest are the model's packing of P."""
    x, want = sweeps["P"], sweeps["P_packed"]
    for pitch, width, phase in ((16, 8, 0), (56, 40, 5)):
        src, off = gathered_source(x, pitch, width, phase)
        out = torch.full((want.size,), 0xA5, dtype=torch.uint8, device="cuda")
        dg, st, _ = _engine.run_fp8([(src.data_ptr() + 2 * off, out.data_ptr(), x.size, None, None, (pitch, width, phase))], False, _stream())
        assert st == [0], (pitch, width)
        check_packed(_host(out), want, x.size, f"gathered pack (pitch {pitch}, width {width}, phase {phase})")
        assert dg == [bb.bbh64(want)], (pitch, width)


GUARD = 0x5A5A


@pytest.mark.gpu
def test_fused_unpack_matches_model(bb, sweeps, _engine):
    """The fused unpack (bb_xfer_fp8 get) of U and of the model's packing of P: the whole object with its expected
    digest, an element window and a strided window, each into a guard-filled buffer."""
    objs = [(sweeps["P_packed"], sweeps["P"].size, sweeps["P_back"])] + [u + (b,) for u, b in zip(sweeps["U"], sweeps["U_back"])]
    for i, (packed, n, back) in enumerate(objs):
        slab, digest = _dev(packed), bb.bbh64(packed)
        lo, hi = 1003, n - 77  # an element window: both ends inside a block, reaching into the last tile
        # a strided window: rows of 40 every 96 elements (phase 88), from element 13, inside a row, to the end
        pitch, width, phase = 96, 40, 88
        y = np.arange(13, n, dtype=np.int64) + phase
        keep = y % pitch < width
        cases = [(None, np.arange(n), np.arange(n)), ((lo, hi), np.arange(lo, hi), np.arange(lo, hi)),
                 ((13, n, pitch, width, phase), (y - phase)[keep], (y // pitch * width + y % pitch)[keep])]
        for win, src_el, dst_el in cases:
            out = torch.full((n + 16,), GUARD, dtype=torch.int16, device="cuda")
            item = (out.data_ptr() + 16, slab.data_ptr(), n, digest) + ((win,) if win else ())
            dg, st, _ = _engine.run_fp8([item], True, _stream())
            assert st == [0] and dg == [digest], (i, win)
            got, expect = _host(out), np.full(n + 16, GUARD, dtype=np.uint16)
            expect[8 + dst_el] = back[src_el]
            same_bits(got, expect, "bf16", f"fused unpack of object {i}, window {win}")


@pytest.mark.gpu
def test_tensor_store_round_trips_match_model(bb, sweeps, cuda):
    """TensorStore.put(..., pack_fp8=True) of P's elements as a contiguous tensor (fused pack), as a narrow view (gathered
    pack) and with a numel that is no multiple of 32 (padded, stand-alone pack), read back with get, get_rows and
    get_slice: every result is the model's dequantisation of the model's packing of the same elements."""
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    P = sweeps["P"]
    R = P.size // 160 * 4  # rows of 40: R * 40 elements, a whole number of blocks
    q = P[:R * 40]
    wide = np.resize(GAP_FILL, (R, 56))
    wide[:, 8:48] = q.reshape(R, 40)
    whole = torch.from_numpy(q.view(np.int16).copy()).cuda().view(torch.bfloat16).view(R, 40)
    big = torch.from_numpy(wide.view(np.int16).copy()).cuda().view(torch.bfloat16)
    forms = {"c": whole, "v": big.narrow(1, 8, 40), "pad": whole[:R - 1]}

    def expected(t):
        x = q[:t.numel()]
        padded = np.concatenate([x, np.zeros(-x.size % 32, dtype=np.uint16)])
        return model_unpack(model_pack(padded), padded.size)[:x.size].reshape(tuple(t.shape))

    cl = GpuRankCluster(slab_bytes=128 << 20, cluster_id="t-mxfp8-exh")
    try:
        store = TensorStore(cl.client)
        assert store._gatherable(forms["v"]) is not None and forms["pad"].numel() % 32 != 0
        for k, t in forms.items():
            store.put(k, t, pack_fp8=True)
            want = expected(t)
            rows = (R // 3, R // 3 + 517)
            got = {"get": store.get(k), "get_rows": store.get_rows(k, *rows), "get_slice": store.get_slice(k, 1, 8, 24)}
            exp = {"get": want, "get_rows": want[rows[0]:rows[1]], "get_slice": want[:, 8:24]}
            for how, g in got.items():
                assert tuple(g.shape) == exp[how].shape, (k, how)
                same_bits(_host(g.contiguous().view(torch.int16)), exp[how], "bf16", f"{k}: {how}")
    finally:
        cl.stop()
