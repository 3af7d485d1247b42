"""MXFP8 packing of fp16 and fp32 tensors, against an exact model, through every implementation: the CPU reference, the
stand-alone kernels, the fused pack (1-3 replicas, gathered) and the fused unpack (whole object, element window, strided
window, scattering store).

The model extends the float64 model of test_mxfp8_exhaustive.py to the wide types of common/mxfp8.h: a block's scale is
clamp(floor(log2 amax) - 8 + 127, 0, 254) of its exact values (NaN skipped; 127 for a zero or Inf amax), each element
is RNE(x * 2^(127 - scale)) on the E4M3 grid, saturated; an unpack rounds the exact product once to fp16 (or not at
all for fp32).  float64 holds every product exactly (24 significant bits at most), so the only roundings are the
format's.  The model is checked against torch's float8_e4m3fn, float16 and float32 conversions on every value it is
used on.

Input sets:
  H  every finite fp16 under the block scale of every fp16 binade, the 10 subnormal binades included (scale bytes
     95..134), the block maximum rotated through the 32 lanes; plus blocks of fp16 specials;
  F  for every fp32 exponent field, blocks of seeded random significands under an anchor of that field; then, under
     the scales of a few binades, every E4M3 rounding tie and the fp32 values just below and above it, and the
     448 / 464 / 480 saturation edge; plus blocks of fp32 specials;
  U  every (E4M3 byte, E8M0 byte) pair (test_mxfp8_exhaustive.unpack_tables), unpacked to fp16 and to fp32.
The consistency rule is checked too: on bf16-representable inputs, packing from fp16 or fp32 gives the bytes (and the
digest) of packing from bf16, and a bf16 unpack is the bf16 rounding of the fp32 unpack."""
import numpy as np
import pytest
import torch

from test_mxfp8_exhaustive import bf16_value, check_packed, e4m3_encode, model_pack, model_products, pack_sweep, same_bits, unpack_tables

T = 16384
NP = {"f16": np.uint16, "f32": np.uint32}
FL = {"f16": np.float16, "f32": np.float32}
SIZE = {"f16": 2, "f32": 4}


def mxw(bb, w):
    return {"bf16": bb.MxWide.BF16, "f16": bb.MxWide.F16, "f32": bb.MxWide.F32}[w]


# ---------------------------------------------------------------------------------------------------- the model


def wide_value(bits, w):
    """float64 value of raw fp16 / fp32 / bf16 patterns (exact)."""
    bits = np.asarray(bits)
    if w == "bf16":
        return bf16_value(bits)
    with np.errstate(invalid="ignore"):
        return bits.astype(NP[w]).view(FL[w]).astype(np.float64)


def model_scales_w(vals):
    """E8M0 byte per 32-element block of exact values: floor(log2 amax) from frexp, so an fp16 subnormal amax gets its
    true binade and an fp32 subnormal amax clamps to 0."""
    a = np.abs(vals.reshape(-1, 32))
    amax = np.where(np.isnan(a), 0.0, a).max(axis=1)
    _, ex = np.frexp(np.where(np.isinf(amax), 1.0, amax))
    e = np.clip(ex - 1 - 8 + 127, 0, 254)
    return np.where((amax == 0) | np.isinf(amax), 127, e).astype(np.uint8)


def model_scaled_w(x, w):
    vals = wide_value(x, w)
    s = model_scales_w(vals)
    return s, (vals.reshape(-1, 32) * np.ldexp(1.0, 127 - s.astype(np.int64))[:, None]).reshape(-1)


def model_pack_w(x, w):
    s, v = model_scaled_w(x, w)
    return np.concatenate([e4m3_encode(v), s])


def f16_encode(v):
    """fp16 patterns of float64 values: RNE onto the grid of step 2^(max(floor(log2|v|), -14) - 10); values at or past
    65520 become +-Inf; NaN -> 0x7E00."""
    nan = np.isnan(v)
    a = np.where(nan, 0.0, np.abs(v))
    _, ex = np.frexp(np.where(np.isinf(a), 0.0, a))
    step = np.ldexp(1.0, np.maximum(ex - 1, -14) - 10)
    q = np.rint(a / step) * step
    q = np.copysign(np.where(q >= 65536.0, np.inf, q), v)
    with np.errstate(over="ignore"):
        bits = np.where(nan, 0.0, q).astype(np.float16).view(np.uint16)
    return np.where(nan, np.uint16(0x7E00), bits)


def model_unpack_w(packed, n, w):
    p = model_products(packed, n)
    if w == "f16":
        return f16_encode(p)
    with np.errstate(over="ignore"):
        return p.astype(np.float32).view(np.uint32)  # exact; +-Inf past fp32 for scale bytes >= 247


def same_wide(got, want, w, what):
    """Bit for bit, the sign of zero included; a NaN only has to be a NaN."""
    got, want = np.asarray(got).reshape(-1).view(NP[w]), np.asarray(want).reshape(-1).view(NP[w])
    assert got.shape == want.shape, f"{what}: {got.shape} elements, want {want.shape}"
    gnan, wnan = np.isnan(got.view(FL[w])), np.isnan(want.view(FL[w]))
    bad = (gnan != wnan) | (~wnan & (got != want))
    if bad.any():
        i = np.nonzero(bad)[0][:8]
        pytest.fail(f"{what}: {int(bad.sum())} of {bad.size} {w} values differ, at {i.tolist()}: "
                    f"got {[hex(v) for v in got[i]]}, want {[hex(v) for v in want[i]]}")


# ---------------------------------------------------------------------------------------------------- the input sets


def _blocks(groups):
    """Blocks of 31 fill elements next to an anchor: groups = [(fill patterns, anchor pattern, sign bit)].  Block j puts
    its anchor at position j % 32 with sign (-1)^(j // 32)."""
    fills, anchors, sign_bit = [], [], None
    for fill, anchor, sb in groups:
        nb = -(-fill.size // 31)
        fills.append(np.resize(fill, nb * 31).reshape(nb, 31))
        anchors.append(np.full(nb, anchor, dtype=fill.dtype))
        sign_bit = sb
    fill, anchor = np.concatenate(fills), np.concatenate(anchors)
    j = np.arange(anchor.size)
    anchor = anchor | (((j >> 5) & 1).astype(anchor.dtype) * anchor.dtype.type(sign_bit))
    at = np.arange(32)[None, :] == (j % 32)[:, None]
    out = np.empty((anchor.size, 32), dtype=anchor.dtype)
    out[at] = anchor
    out[~at] = fill.reshape(-1)
    return out.reshape(-1)


def f16_sweep():
    """H: for every fp16 binade [2^k, 2^(k+1)), k = -24..15, every finite fp16 x with |x| < 2^(k+1), half of the ones at
    most 2^k next to the anchor 2^k and the rest next to the anchor top(k), the largest fp16 below 2^(k+1)."""
    rng = np.random.default_rng(1)
    groups = []
    for k in range(-24, 16):
        low = (k + 15) << 10 if k >= -14 else 1 << (k + 24)
        top = ((k + 16) << 10 if k >= -15 else 1 << (k + 25)) - 1
        mags = np.arange(top + 1, dtype=np.uint16)
        xs = np.concatenate([mags, mags | 0x8000])
        rng.shuffle(xs)
        under = (xs & 0x7FFF) <= low
        kk = int(under.sum()) // 2
        lo_set = xs[under][:kk]
        hi_set = xs[~(under & (np.cumsum(under) <= kk))]
        groups += [(hi_set, top, 0x8000), (lo_set, low, 0x8000)]
    return _blocks([g for g in groups if g[0].size])


def f16_specials():
    """Blocks of fp16 NaN (both signs, several payloads), +-Inf, +-0 and subnormals around a maximum at each position."""
    rows = []
    for p in range(32):
        m = ((2 + p * 28 // 31) << 10) | (p * 37 % 1024)  # exponent fields 2..30
        fill = np.array([0x0000, 0x8000, 0x0001, 0x8001, 0x03FF, 0x83FF, 0x7E00, 0xFE01, 0x7C01, 0xFFFF]
                        + [(m - k * 0x53) | (0x8000 if k % 2 else 0) for k in range(1, 22)], dtype=np.uint16)
        fill = np.roll(fill, 3 * p)
        rows += [np.insert(fill, p, v) for v in (m, m | 0x8000, 0x7C00, 0xFC00, 0x7E00, 0x7C01)]
        rows.append(np.insert(np.resize(np.array([0x7E00, 0xFE01, 0x7FFF], dtype=np.uint16), 31), p, 0x7C01))  # all NaN
        rows.append(np.insert(np.resize(np.array([0x0000, 0x8000], dtype=np.uint16), 31), p, 0x8000))  # all zero
        rows.append(np.insert(np.arange(1, 32, dtype=np.uint16) * 3, p, 0x83FF))  # subnormals only
    return np.concatenate(rows)


def e4m3_grid():
    """The positive finite E4M3 values, ascending (0 first)."""
    b = np.arange(0x7F, dtype=np.uint8)
    e, m = (b >> 3) & 15, b & 7
    return np.where(e == 0, m * 2.0 ** -9, np.ldexp(1.0 + m / 8.0, e.astype(np.int64) - 7))


def f32_sweep():
    """F: random-significand blocks under an anchor of every exponent field, then the tie set."""
    rng = np.random.default_rng(2)
    groups = []
    for f in range(255):
        for rep in range(2):
            anchor = (f << 23) | int(rng.integers(0, 1 << 23))
            fields = rng.integers(0, f + 1, 31 * 20, dtype=np.uint32)
            fill = (fields << 23) | rng.integers(0, 1 << 23, fields.size, dtype=np.uint32)
            fill = np.minimum(fill, np.uint32(anchor)) | (rng.integers(0, 2, fill.size, dtype=np.uint32) << 31)
            groups.append((fill.astype(np.uint32), anchor, 0x80000000))
    # ties: under the scale of an anchor 2^(8 + k) every value x * 2^k with x at, just below and just above each midpoint
    # of two neighbouring E4M3 values (0 and 2^-9 included), and the saturation edge
    g = e4m3_grid()
    mids = ((g[:-1] + g[1:]) / 2).astype(np.float32)
    ties = np.concatenate([mids, np.nextafter(mids, np.float32(0)), np.nextafter(mids, np.float32(np.inf)),
                           np.array([448.0, 456.0, 463.99997, 464.0, 464.00003, 480.0, 500.0, 511.99997], dtype=np.float32)])
    for k in (-110, -40, 0, 25, 100):
        vals = (ties.astype(np.float64) * 2.0 ** k).astype(np.float32)
        assert np.array_equal(vals.astype(np.float64), ties.astype(np.float64) * 2.0 ** k)  # exact in fp32
        anchor = np.float32(2.0 ** (8 + k)).view(np.uint32)
        bits = vals.view(np.uint32)
        groups.append((np.concatenate([bits, bits | np.uint32(0x80000000)]), int(anchor), 0x80000000))
    return _blocks(groups)


def f32_specials():
    rows = []
    for p in range(32):
        m = np.float32(2.0 ** (p * 7 - 100) * (1 + p / 32)).view(np.uint32)
        fill = np.array([0, 0x80000000, 1, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00800000, 0x7FC00000, 0xFFC00001, 0x7F800001]
                        + [(int(m) - k * 0x12345) | (0x80000000 if k % 2 else 0) for k in range(1, 22)], dtype=np.uint32)
        fill = np.roll(fill, 3 * p)
        rows += [np.insert(fill, p, v) for v in (m, m | 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0x7F7FFFFF)]
        rows.append(np.insert(np.resize(np.array([0x7FC00000, 0xFFC00001], dtype=np.uint32), 31), p, 0x7F800001))
        rows.append(np.insert(np.arange(1, 32, dtype=np.uint32) * 7, p, 0x807FFFFF))  # fp32 subnormals only
    return np.concatenate(rows)


@pytest.fixture(scope="module")
def sets():
    x = {"f16": np.concatenate([f16_sweep(), f16_specials()]), "f32": np.concatenate([f32_sweep(), f32_specials()])}
    packed = {w: model_pack_w(v, w) for w, v in x.items()}
    U = unpack_tables()
    back = {w: [model_unpack_w(u, n, w) for u, n in U] for w in ("f16", "f32")}
    return {"x": x, "packed": packed, "U": U, "U_back": back}


# ---------------------------------------------------------------------------------------------------- CPU


def test_sets_reach_every_binade(sets):
    """H reaches scale bytes 95..134 (fp16's ten subnormal binades included); F reaches 0..246 and every tie."""
    x, p = sets["x"], sets["packed"]
    n16 = x["f16"].size
    s16 = np.unique(p["f16"][n16:])
    assert np.array_equal(s16, np.arange(95, 135)), s16
    n32 = x["f32"].size
    assert np.array_equal(np.unique(p["f32"][n32:]), np.arange(247))
    assert n16 % 32 == 0 and n32 % 32 == 0


def test_model_matches_torch(sets):
    """E4M3 of the scaled elements vs torch float8_e4m3fn; the fp16 and fp32 roundings of the unpacked products vs
    torch's float16 / float32 conversions."""
    for w in ("f16", "f32"):
        _, v = model_scaled_w(sets["x"][w], w)
        # every scaled value is exact in fp32, or below 2^-126 (and so +-0 in E4M3 either way)
        ref = torch.from_numpy(v.astype(np.float32)).clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8).numpy()
        same_bits(e4m3_encode(v), ref, "e4m3", f"{w}: E4M3 vs torch")
        objs = [(sets["packed"][w], sets["x"][w].size)] + sets["U"]
        for i, (packed, m) in enumerate(objs):
            prod = model_products(packed, m).astype(np.float32)  # exact: at most 4 significant bits, >= 2^-136
            want = model_unpack_w(packed, m, w)
            dt = torch.float16 if w == "f16" else torch.float32
            ref = torch.from_numpy(prod).to(dt).numpy().view(NP[w])
            same_wide(want, ref, w, f"{w}: object {i} vs torch")


def test_cpu_reference_matches_model(bb, sets):
    for w in ("f16", "f32"):
        x = sets["x"][w]
        got = np.frombuffer(bb.mxfp8_pack_ref(x, mxw(bb, w)), dtype=np.uint8)
        check_packed(got, sets["packed"][w], x.size, f"mxfp8_pack_ref({w})")
        for i, ((u, m), back) in enumerate(zip(sets["U"], sets["U_back"][w])):
            same_wide(np.frombuffer(bb.mxfp8_unpack_ref(u, m, mxw(bb, w)), dtype=NP[w]), back, w, f"mxfp8_unpack_ref(U{i}, {w})")


def test_e4m3_from_float_on_full_significands(bb, sets):
    """The CPU E4M3 rounding on full 24-bit significands: every distinct scaled value of F, ties included."""
    _, v = model_scaled_w(sets["x"]["f32"], "f32")
    v = np.unique(v.astype(np.float32).view(np.uint32)).view(np.float32)
    got = np.array([bb.e4m3_from_float(float(f)) for f in v], dtype=np.uint8)
    same_bits(got, e4m3_encode(v.astype(np.float64)), "e4m3", "e4m3_from_float on F")


@pytest.fixture(scope="module")
def consistent():
    """bf16-representable inputs: the exhaustive bf16 sweep as bf16 and as fp32 bits; and H rounded to bf16 (a value that
    then leaves fp16's range, 65504 -> 65536, becomes 0) as fp16 and as bf16 bits."""
    P = pack_sweep()
    h = torch.from_numpy(np.concatenate([f16_sweep(), f16_specials()]).view(np.int16).copy()).view(torch.float16)
    hb = h.float().to(torch.bfloat16)
    hb = torch.where(hb.float().abs() > 65504, torch.zeros_like(hb), hb)
    return {"bf16": P, "f32": (P.astype(np.uint32) << 16), "bf16_16": hb.view(torch.int16).numpy().view(np.uint16),
            "f16": hb.float().half().view(torch.int16).numpy().view(np.uint16)}


def test_consistency_cpu(bb, consistent):
    """pack(F32) and pack(F16) of bf16-representable inputs are pack(BF16); unpack(BF16) is bf16(unpack(F32))."""
    c = consistent
    ref = bb.mxfp8_pack_ref(c["bf16"])
    assert bb.mxfp8_pack_ref(c["f32"], bb.MxWide.F32) == ref
    assert bb.mxfp8_pack_ref(c["f16"], bb.MxWide.F16) == bb.mxfp8_pack_ref(c["bf16_16"])
    assert np.array_equal(wide_value(c["f16"], "f16"), bf16_value(c["bf16_16"]), equal_nan=True)
    for u, m in unpack_tables():
        b = np.frombuffer(bb.mxfp8_unpack_ref(u, m), dtype=np.uint16)
        f = np.frombuffer(bb.mxfp8_unpack_ref(u, m, bb.MxWide.F32), dtype=np.float32)
        want = torch.from_numpy(f.copy()).to(torch.bfloat16).view(torch.int16).numpy()
        same_bits(b, want, "bf16", "unpack(BF16) vs bf16(unpack(F32))")


# ---------------------------------------------------------------------------------------------------- GPU


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()


def _host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need CUDA (marked gpu)")


@pytest.fixture(scope="module")
def engine(cuda):
    from blackbird_b200 import _bb

    return _bb.XferEngine(0, 4096, 2)


@pytest.mark.gpu
def test_standalone_kernels_match_model(bb, sets, cuda):
    for w in ("f16", "f32"):
        x, n = sets["x"][w], sets["x"][w].size
        out = torch.empty(bb.mxfp8_packed_bytes(n), dtype=torch.uint8, device="cuda")
        bb.mxfp8_pack(_dev(x).data_ptr(), n, out.data_ptr(), _stream(), wide=mxw(bb, w))
        check_packed(_host(out), sets["packed"][w], n, f"mxfp8_pack({w})")
        for i, ((u, m), back) in enumerate(zip(sets["U"], sets["U_back"][w])):
            o = torch.empty(m * SIZE[w], dtype=torch.uint8, device="cuda")
            bb.mxfp8_unpack(_dev(u).data_ptr(), m, o.data_ptr(), _stream(), wide=mxw(bb, w))
            same_wide(_host(o), back, w, f"mxfp8_unpack(U{i}, {w})")


def gathered(x, w, pitch, width, phase):
    """x as rows of `width` elements every `pitch`, row 0 starting `phase` elements before x[0] at a 16-byte aligned
    address; the gaps hold NaN, +-Inf and +-max of the type.  Returns (device buffer, pointer offset in elements)."""
    fill = {"f16": [0x7E00, 0xFC00, 0x7BFF, 0x7C00, 0xFBFF], "f32": [0x7FC00000, 0xFF800000, 0x7F7FFFFF, 0x7F800000, 0xFF7FFFFF]}[w]
    per = 16 // SIZE[w]
    y = np.arange(x.size, dtype=np.int64) + phase
    idx = y // width * pitch + y % width
    off = (per - phase % per) % per
    buf = np.resize(np.array(fill, dtype=NP[w]), off + int(idx[-1]) + 1 + 64)
    buf[off + idx] = x
    return _dev(buf), off


@pytest.mark.gpu
def test_fused_pack_matches_model(bb, sets, engine):
    """The fused pack into 1, 2 and 3 replicas, and gathered from rows whose gaps hold NaN / Inf / max; every replica
    holds the model's packing and the digest is bbh64 of it."""
    for w in ("f16", "f32"):
        x, want = sets["x"][w], sets["packed"][w]
        src = _dev(x)
        for nrep in (1, 2, 3):
            reps = [torch.full((want.size,), 0xA5, dtype=torch.uint8, device="cuda") for _ in range(nrep)]
            dg, st, _ = engine.run_fp8([(src.data_ptr(), [r.data_ptr() for r in reps], x.size)], False, _stream(), wide=mxw(bb, w))
            assert st == [0] and dg == [bb.bbh64(want)], (w, nrep)
            for r in reps:
                check_packed(_host(r), want, x.size, f"fused pack({w}, {nrep} replicas)")
        per = 16 // SIZE[w]
        for pitch, width, phase in ((2 * per, per, 0), (7 * per, 5 * per, 3)):
            g, off = gathered(x, w, pitch, width, phase)
            out = torch.full((want.size,), 0xA5, dtype=torch.uint8, device="cuda")
            dg, st, _ = engine.run_fp8([(g.data_ptr() + SIZE[w] * off, out.data_ptr(), x.size, None, None, (pitch, width, phase))], False,
                                       _stream(), wide=mxw(bb, w))
            assert st == [0] and dg == [bb.bbh64(want)], (w, pitch, width)
            check_packed(_host(out), want, x.size, f"gathered pack({w}, pitch {pitch}, width {width}, phase {phase})")


@pytest.mark.gpu
def test_fused_unpack_matches_model(bb, sets, engine):
    """The fused unpack of U and of the model's packing of H / F to fp16 and fp32: whole, an element window, a strided
    window and a scattering store, each into a guard-filled buffer."""
    for w in ("f16", "f32"):
        b, per = SIZE[w], 16 // SIZE[w]
        guard = NP[w](0x5A5A5A5A & ((1 << (8 * b)) - 1))
        objs = [(sets["packed"][w], sets["x"][w].size)] + sets["U"]
        for i, (packed, n) in enumerate(objs):
            back = model_unpack_w(packed, n, w)
            slab, digest = _dev(packed), bb.bbh64(packed)
            lo, hi = 1003, n - 77
            pitch, width, phase = 24 * per, 10 * per, 22 * per
            y = np.arange(13, n, dtype=np.int64) + phase
            keep = y % pitch < width
            cases = [(None, np.arange(n), np.arange(n)), ((lo, hi), np.arange(lo, hi), np.arange(lo, hi)),
                     ((13, n, pitch, width, phase), (y - phase)[keep], (y // pitch * width + y % pitch)[keep])]
            for win, src_el, dst_el in cases:
                out = torch.from_numpy(np.full(n + 2 * per, guard, dtype=NP[w]).view(np.uint8).copy()).cuda()
                item = (out.data_ptr() + 16, slab.data_ptr(), n, digest) + ((win,) if win else ())
                dg, st, _ = engine.run_fp8([item], True, _stream(), wide=mxw(bb, w))
                assert st == [0] and dg == [digest], (w, i, win)
                expect = np.full(n + 2 * per, guard, dtype=NP[w])
                expect[per + dst_el] = back[src_el]
                same_wide(_host(out), expect, w, f"fused unpack({w}) of object {i}, window {win}")
            # scattering store: rows of 5 * per elements every 7 * per, phase 3
            sp, sw, sph = 7 * per, 5 * per, 3
            yy = np.arange(n, dtype=np.int64) + sph
            at = yy // sw * sp + yy % sw
            off = (per - sph % per) % per
            out = torch.from_numpy(np.full(off + int(at[-1]) + 1 + per, guard, dtype=NP[w]).view(np.uint8).copy()).cuda()
            dg, st, _ = engine.run_fp8([(out.data_ptr() + b * off, slab.data_ptr(), n, digest, None, None, (sp, sw, sph))], True, _stream(),
                                       wide=mxw(bb, w))
            assert st == [0] and dg == [digest], (w, i, "scatter")
            expect = np.full(off + int(at[-1]) + 1 + per, guard, dtype=NP[w])
            expect[off + at] = back
            same_wide(_host(out), expect, w, f"fused scattered unpack({w}) of object {i}")


@pytest.mark.gpu
def test_fused_consistency(bb, consistent, engine):
    """On bf16-representable inputs the fused pack from fp16 / fp32 stores the bytes and digest of the bf16 pack, and
    the fused bf16 unpack of every (payload, scale) pair is the bf16 rounding of the fused fp32 unpack."""
    c = consistent
    for w, key, ref_key in (("f32", "f32", "bf16"), ("f16", "f16", "bf16_16")):
        n = c[key].size
        outs = {}
        for ww, k in ((w, key), ("bf16", ref_key)):
            src = _dev(c[k])
            out = torch.empty(bb.mxfp8_packed_bytes(n), dtype=torch.uint8, device="cuda")
            dg, st, _ = engine.run_fp8([(src.data_ptr(), out.data_ptr(), n)], False, _stream(), wide=mxw(bb, ww))
            assert st == [0]
            outs[ww] = (_host(out), dg[0])
        assert np.array_equal(outs[w][0], outs["bf16"][0]) and outs[w][1] == outs["bf16"][1], w
    for u, m in unpack_tables():
        slab = _dev(u)
        o32 = torch.empty(m, dtype=torch.float32, device="cuda")
        o16 = torch.empty(m, dtype=torch.bfloat16, device="cuda")
        engine.run_fp8([(o32.data_ptr(), slab.data_ptr(), m)], True, _stream(), wide=bb.MxWide.F32)
        engine.run_fp8([(o16.data_ptr(), slab.data_ptr(), m)], True, _stream())
        same_bits(_host(o16.view(torch.int16)), _host(o32.to(torch.bfloat16).view(torch.int16)), "bf16", "bf16 unpack vs bf16(fp32 unpack)")


@pytest.mark.gpu
def test_mixed_batches(bb, engine):
    """A batch of bf16 and fp16 items (the type per item) takes the launches of a bf16-only batch, and each item is
    packed and unpacked by its own type; a batch that mixes 2- and 4-byte items is INVALID_ARGUMENT and launches
    nothing."""
    n = 4 * T + 96
    x = torch.randn(2, n, device="cuda") * 3
    a16, ab, a32 = x[0].half(), x[1].bfloat16(), x[0].float()
    outs = [torch.empty(bb.mxfp8_packed_bytes(n), dtype=torch.uint8, device="cuda") for _ in range(2)]
    before = engine.launches
    engine.run_fp8([(ab.data_ptr(), outs[0].data_ptr(), n), (ab.data_ptr(), outs[1].data_ptr(), n)], False, _stream())
    per_batch = engine.launches - before
    before = engine.launches
    dg, st, _ = engine.run_fp8([(ab.data_ptr(), outs[0].data_ptr(), n, None, None, None, None, bb.MxWide.BF16),
                                (a16.data_ptr(), outs[1].data_ptr(), n, None, None, None, None, bb.MxWide.F16)], False, _stream())
    assert engine.launches - before == per_batch and st == [0, 0]
    want = [model_pack_w(_host(ab.view(torch.int16)).view(np.uint16), "bf16"), model_pack_w(_host(a16.view(torch.int16)).view(np.uint16), "f16")]
    for o, wnt, d in zip(outs, want, dg):
        check_packed(_host(o), wnt, n, "mixed batch pack")
        assert d == bb.bbh64(wnt)
    backs = [torch.empty(n, dtype=torch.bfloat16, device="cuda"), torch.empty(n, dtype=torch.float16, device="cuda")]
    before = engine.launches
    dg, st, _ = engine.run_fp8([(backs[0].data_ptr(), outs[0].data_ptr(), n, None, None, None, None, bb.MxWide.BF16),
                                (backs[1].data_ptr(), outs[1].data_ptr(), n, None, None, None, None, bb.MxWide.F16)], True, _stream())
    assert engine.launches - before == per_batch and st == [0, 0]
    same_bits(_host(backs[0].view(torch.int16)), bf16_of(want[0], n), "bf16", "mixed bf16 unpack")
    same_wide(_host(backs[1].view(torch.int16)), model_unpack_w(want[1], n, "f16"), "f16", "mixed f16 unpack")
    before = engine.launches
    with pytest.raises(RuntimeError, match="INVALID_ARGUMENT"):
        engine.run_fp8([(ab.data_ptr(), outs[0].data_ptr(), n), (a32.data_ptr(), outs[1].data_ptr(), n, None, None, None, None, bb.MxWide.F32)],
                       False, _stream())
    assert engine.launches == before


def bf16_of(packed, n):
    from test_mxfp8_exhaustive import model_unpack

    return model_unpack(packed, n)
