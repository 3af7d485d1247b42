"""Paged puts and gets of MXFP8-packed tensors (batch_put_device_fp8_paged, batch_get_device_fp8_paged) on CPU: the
HostLoopbackTransport stands in for the GPU fabric and runs the CPU codec, so the client's rules in element units -- the
table in wide bytes, co-alignment, whole MX blocks, the refusals, replica fan-out, fail-over and the placement refresh --
run in the CPU suite under the same SourcePages rule the kernels follow.  Page addresses here are host addresses: the
loopback's "device pointers" are host pointers."""
import numpy as np

from blackbird_b200.parallel import LocalCluster

MiB = 1 << 20
T = 16384
GUARD = 0xA5
NP = {"bf16": np.uint16, "f16": np.float16, "f32": np.float32}
SIZE = {"bf16": 2, "f16": 2, "f32": 4}


def mxw(bb, w):
    return {"bf16": bb.MxWide.BF16, "f16": bb.MxWide.F16, "f32": bb.MxWide.F32}[w]


def make_client(bb, c, node="node-0"):
    cl = c.client(node_id=node)
    io = c.client(node_id=node)
    bb.attach_loopback_transport(cl, io, False)
    return cl


def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


def _cfg(bb, replicas):
    return bb.WorkerConfig(replication_factor=replicas, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_CPU])


def _sums(cl, key):
    return [[sh.checksum for sh in cp.shards] for cp in cl.get_workers(key)]


def _values(rng, n, w):
    """n elements of type w over many binades, with a few specials, as raw bytes."""
    v = (rng.standard_normal(n) * np.exp2(rng.integers(-12, 12, n))).astype(np.float32)
    v[::97] = np.nan
    v[7::331] = 0.0
    x = v.astype(NP[w]) if w != "bf16" else (v.view(np.uint32) >> 16).astype(np.uint16)
    return x.view(np.uint8)


class Arena:
    """One guard-filled host buffer that pages are carved from: 16-byte aligned plus a chosen skew, with a guard gap
    after every page."""

    def __init__(self, nbytes):
        self.raw = np.full(nbytes, GUARD, dtype=np.uint8)
        self.base = self.raw.ctypes.data
        self.o = (-self.base) % 16 + 64

    def pages(self, n, page, skew=0, shuffle=None):
        offs = []
        for _ in range(n):
            offs.append(self.o + skew)
            self.o = (self.o + skew + page + 15) // 16 * 16 + 48
        assert self.o < len(self.raw)
        if shuffle is not None:
            offs = [offs[i] for i in shuffle.permutation(n)]
        return offs

    def addrs(self, offs):
        return np.array([self.base + o for o in offs], dtype=np.uint64)

    def fill(self, offs, page, blob):
        for k, o in enumerate(offs):
            self.raw[o:o + page] = blob[k * page:(k + 1) * page]

    def expect(self, offs, page, blob):
        """The whole buffer as it must be: guard everywhere except blob cut into the pages."""
        want = np.full_like(self.raw, GUARD)
        for k, o in enumerate(offs):
            want[o:o + page] = blob[k * page:(k + 1) * page]
        return want


# ---------------------------------------------------------------- the rule in element units against a numpy model
def test_to_wide_bytes_and_the_element_rule_match_the_numpy_model(bb):
    rng = np.random.default_rng(11)
    for _ in range(300):
        b = int(rng.choice([2, 4]))
        npages = int(rng.integers(1, 20))
        pe = int(rng.choice([1, 3, 8, 12, 24, 100, 4096]))
        base = int(rng.integers(0, 1 << 40)) * 16
        addrs = [base + int(o) * pe * b + (int(rng.integers(0, 8)) * 2 if rng.random() < 0.2 else 0) for o in rng.permutation(npages)]
        ec, t, n = bb.SourcePages.from_pages(addrs, pe)
        assert ec == bb.ErrorCode.OK and n == npages * pe
        off = int(rng.integers(0, n + 1))
        r = t.rebase(off)
        ok, w = r.to_wide_bytes(b)
        assert ok and (w.page, w.phase, w.addrs, w.npages) == (pe * b, r.phase * b, r.addrs, r.npages)
        # element x of the element table lives where byte b * x of the wide-byte table does
        m = n - off
        xs = np.arange(m)
        k0 = min(off // pe, npages)
        want = np.asarray(addrs[k0:], dtype=np.int64)[(xs + off % pe) // pe] + b * ((xs + off % pe) % pe) if m else xs
        got = [a + j for x0, a, cnt in w.runs(b * m) for j in range(0, cnt, b)]
        assert got == list(want)
        # co-alignment in wide bytes: every page touched at addrs[k] + b * phase 16-byte aligned, b * pe % 16 == 0 for several
        touched = (m - 1 + off % pe) // pe + 1 if m else 0
        model = (touched <= 1 or (b * pe) % 16 == 0) and all((a + b * (off % pe)) % 16 == 0 for a in addrs[k0:k0 + touched])
        assert w.coaligned(b * m) == model
    # overflow of page or phase in wide bytes
    _, t, _ = bb.SourcePages.from_pages([16], 1 << 63)
    assert t.to_wide_bytes(2)[0] is False and t.to_wide_bytes(1)[0] is True
    _, t, _ = bb.SourcePages.from_pages([16], (1 << 62) + 1)
    assert t.to_wide_bytes(4)[0] is False and t.to_wide_bytes(2)[0] is True


# ---------------------------------------------------------------- client calls through the loopback transport
# (page elements, pages, skew in elements): pages that are not a multiple of 32 elements (MX blocks straddle pages), one
# page, pages longer than a tile
def _shapes(w):
    per = 16 // SIZE[w]
    return [(3 * per, 96, 0), (5 * per, 64, 0), (T, 1, 0), (T + 32 * per, 3, 0), (64 * per, 7, 0)]


def test_put_equals_a_packed_put_of_the_concatenation(bb):
    """Shuffled pages with guard gaps, for bf16, fp16 and fp32: the stored bytes are the reference packing of the
    concatenation, the digests those of batch_put_device_fp8 of it, and both read back through plain and paged gets."""
    rng = np.random.default_rng(12)
    with LocalCluster(cluster_id="fp8pg", n_workers=2, pool_bytes=96 * MiB) as c:
        cl = make_client(bb, c)
        n0 = _counter(cl, "device_put_fp8_paged_total")
        for w in ("bf16", "f16", "f32"):
            b, wd = SIZE[w], mxw(bb, w)
            shapes = _shapes(w)
            ar = Arena(sum(pe * b * n + 64 * n for pe, n, _ in shapes) + MiB)
            keys, tables, blobs, offs_all = [], [], [], []
            for j, (pe, n, _) in enumerate(shapes):
                assert (pe * n) % 32 == 0
                offs = ar.pages(n, pe * b, shuffle=rng)
                blob = _values(rng, pe * n, w)
                ar.fill(offs, pe * b, blob)
                keys.append(f"{w}/{j}"), tables.append(ar.addrs(offs)), blobs.append(blob), offs_all.append(offs)
            before = ar.raw.copy()
            ecs = cl.batch_put_device_fp8_paged(keys, tables, [s[0] for s in shapes], _cfg(bb, 2), 0, wide=wd)
            assert ecs == [bb.ErrorCode.OK] * len(shapes), (w, ecs)
            assert np.array_equal(ar.raw, before)  # a put reads only
            for (ec, stored), blob, key in zip(cl.batch_get(keys), blobs, keys):
                assert ec == bb.ErrorCode.OK and bytes(stored) == bb.mxfp8_pack_ref(blob.view(NP[w]), wd), key
                assert len(cl.get_workers(key)) == 2
            refs = [k + "/ref" for k in keys]
            assert cl.batch_put_device_fp8(refs, [x.ctypes.data for x in blobs], [x.size // b for x in blobs], _cfg(bb, 2), 0,
                                           wide=wd) == [bb.ErrorCode.OK] * len(shapes)
            for k, r in zip(keys, refs):
                assert _sums(cl, k) == _sums(cl, r), k
            for j, (pe, n, _) in enumerate(shapes):
                unpacked = np.frombuffer(bb.mxfp8_unpack_ref(bb.mxfp8_pack_ref(blobs[j].view(NP[w]), wd), pe * n, wd), dtype=np.uint8)
                # a plain fp8 get of the paged object
                out = np.zeros(pe * n * b, np.uint8)
                assert cl.batch_get_device_fp8([keys[j]], [out.ctypes.data], [pe * n], 0, wide=wd) == [bb.ErrorCode.OK]
                assert np.array_equal(out, unpacked), (w, j)
                # a paged get of the plain object into fresh shuffled pages: the pages hold it, every guard byte stays
                dst = Arena(pe * b * n + 64 * n + 4096)
                doffs = dst.pages(n, pe * b, shuffle=rng)
                assert cl.batch_get_device_fp8_paged([refs[j]], [dst.addrs(doffs)], [pe], 0, wide=wd) == [bb.ErrorCode.OK]
                assert np.array_equal(dst.raw, dst.expect(doffs, pe * b, unpacked)), (w, j)
        assert _counter(cl, "device_put_fp8_paged_total") == n0 + 3 * 5
        assert _counter(cl, "device_get_fp8_paged_total") > 0 and _counter(cl, "device_get_fp8_paged_bytes_total") > 0


def test_any_packed_object_reads_into_pages_of_any_wide_type(bb):
    """An fp32 object put from pages reads into bf16 pages (and back), as any packed object reads into any type."""
    rng = np.random.default_rng(13)
    with LocalCluster(cluster_id="fp8pgx", n_workers=1, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        pe, n = 96, 24
        src = Arena(pe * 4 * n + 64 * n + 4096)
        offs = src.pages(n, pe * 4, shuffle=rng)
        blob = _values(rng, pe * n, "f32")
        src.fill(offs, pe * 4, blob)
        assert cl.batch_put_device_fp8_paged(["x"], [src.addrs(offs)], [pe], _cfg(bb, 1), 0, wide=bb.MxWide.F32) == [bb.ErrorCode.OK]
        dst = Arena(pe * 2 * n + 64 * n + 4096)
        doffs = dst.pages(n, pe * 2, shuffle=rng)
        assert cl.batch_get_device_fp8_paged(["x"], [dst.addrs(doffs)], [pe], 0, wide=bb.MxWide.BF16) == [bb.ErrorCode.OK]
        want = np.frombuffer(bb.mxfp8_unpack_ref(bb.mxfp8_pack_ref(blob.view(np.float32), bb.MxWide.F32), pe * n, bb.MxWide.BF16), np.uint8)
        assert np.array_equal(dst.raw, dst.expect(doffs, pe * 2, want))


def test_refusals_fail_alone(bb):
    """Every refusal gives its per-object code before anything is allocated (puts) or read, while the rest of the batch
    succeeds; nothing is written outside the accepted items' pages."""
    rng = np.random.default_rng(14)
    E = bb.ErrorCode
    with LocalCluster(cluster_id="fp8pgr", n_workers=1, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        ar = Arena(4 * MiB)
        good = ar.pages(8, 64 * 2)
        blob = _values(rng, 64 * 8, "bf16")
        ar.fill(good, 128, blob)
        skewed = ar.pages(8, 128, skew=2)   # one element off 16-byte alignment
        odd = ar.pages(8, 36 * 2)           # 72-byte pages: 2 * 36 % 16 != 0, 288 elements = 9 blocks
        short = ar.pages(1, 48)             # 24 elements: not a whole MX block
        tabs = [ar.addrs(good), ar.addrs(good), ar.addrs(short), ar.addrs(good[:2]), ar.addrs(skewed), ar.addrs(odd), ar.addrs(good)]
        pes = [64, 0, 24, 1 << 62, 64, 36, 64]
        keys = ["ok", "zero", "part", "ovf", "skew", "odd", "ok2"]
        ecs = cl.batch_put_device_fp8_paged(keys, tabs, pes, _cfg(bb, 1), 0)
        assert ecs == [E.OK, E.INVALID_ARGUMENT, E.INVALID_ARGUMENT, E.VALUE_OUT_OF_RANGE, E.NOT_IMPLEMENTED, E.NOT_IMPLEMENTED, E.OK]
        for k in ("zero", "part", "ovf", "skew", "odd"):
            assert not cl.object_exists(k), k
        # fp32: 4-element pages are co-aligned (16 bytes), so the same 16-byte rule is % 4 elements there
        f32 = ar.pages(8, 4 * 4)
        assert cl.batch_put_device_fp8_paged(["f32"], [ar.addrs(f32)], [4], _cfg(bb, 1), 0, wide=bb.MxWide.F32) == [E.OK]
        # gets: size mismatch, zero page, not whole blocks, overflow, misaligned, b * page % 16 != 0, missing key, OK
        dst = Arena(4 * MiB)
        d8, d16 = dst.pages(8, 128), dst.pages(16, 128)
        dskew, dodd = dst.pages(8, 128, skew=2), dst.pages(128, 8)  # dodd: 4-element (8-byte) pages
        snapshot = dst.raw.copy()
        ecs = cl.batch_get_device_fp8_paged(
            ["ok", "ok", "ok", "ok", "ok", "ok", "nope", "ok2"],
            [dst.addrs(d16), dst.addrs(d8), dst.addrs(d8[:1]), dst.addrs(d8[:2]), dst.addrs(dskew), dst.addrs(dodd), dst.addrs(d8),
             dst.addrs(d8)],
            [64, 0, 24, 1 << 62, 64, 4, 64, 64], 0)
        assert ecs == [E.INVALID_ARGUMENT, E.INVALID_ARGUMENT, E.INVALID_ARGUMENT, E.VALUE_OUT_OF_RANGE, E.NOT_IMPLEMENTED,
                       E.NOT_IMPLEMENTED, E.OBJECT_NOT_FOUND, E.OK], ecs
        want = np.frombuffer(bb.mxfp8_unpack_ref(bb.mxfp8_pack_ref(blob.view(np.uint16)), blob.size // 2), np.uint8)
        for k, o in enumerate(d8):
            snapshot[o:o + 128] = want[k * 128:(k + 1) * 128]
        assert np.array_equal(dst.raw, snapshot)
        # arity
        assert cl.batch_put_device_fp8_paged(["a", "b"], [[]], [16], _cfg(bb, 1), 0) == [E.INVALID_PARAMETERS] * 2
        assert cl.batch_get_device_fp8_paged(["a", "b"], [[], []], [16], 0) == [E.INVALID_PARAMETERS] * 2


def test_fail_over_and_refresh(bb):
    """A corrupt copy fails the paged get over to the next replica, pages right and guards untouched; with every copy
    corrupt the object is re-read once (placement refresh) and the answer is CHECKSUM_MISMATCH."""
    rng = np.random.default_rng(15)
    with LocalCluster(cluster_id="fp8pgf", n_workers=3, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        pools = {p.id: p for p in cl.keystone().get_memory_pools()}

        def flip(sh, pos):
            wk = [wk for wk in c.workers if wk.backend(sh.pool_id) is not None][0]
            off = sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr + pos
            be = wk.backend(sh.pool_id)
            be.write(off, bytes([be.read(off, 1)[0] ^ 0xFF]))

        pe, n = 2048 + 24, 32  # 4144-byte fp16 pages: MX blocks straddle every page boundary
        src = Arena(pe * 2 * n + 64 * n + 4096)
        offs = src.pages(n, pe * 2, shuffle=rng)
        blob = _values(rng, pe * n, "f16")
        src.fill(offs, pe * 2, blob)
        assert cl.batch_put_device_fp8_paged(["f"], [src.addrs(offs)], [pe], _cfg(bb, 3), 0, wide=bb.MxWide.F16) == [bb.ErrorCode.OK]
        want = np.frombuffer(bb.mxfp8_unpack_ref(bb.mxfp8_pack_ref(blob.view(np.float16), bb.MxWide.F16), pe * n, bb.MxWide.F16), np.uint8)
        copies = cl.get_workers("f")
        assert len(copies) == 3
        fo = _counter(cl, "replica_failover_total")
        for cp in copies:
            flip(cp.shards[0], 4321)
            dst = Arena(pe * 2 * n + 64 * n + 4096)
            doffs = dst.pages(n, pe * 2, shuffle=rng)
            assert cl.batch_get_device_fp8_paged(["f"], [dst.addrs(doffs)], [pe], 0, wide=bb.MxWide.F16) == [bb.ErrorCode.OK]
            assert np.array_equal(dst.raw, dst.expect(doffs, pe * 2, want))
            flip(cp.shards[0], 4321)
        assert _counter(cl, "replica_failover_total") > fo
        for cp in copies:
            flip(cp.shards[0], 7)
        ref = _counter(cl, "get_placement_refresh_total")
        dst = Arena(pe * 2 * n + 64 * n + 4096)
        doffs = dst.pages(n, pe * 2)
        assert cl.batch_get_device_fp8_paged(["f"], [dst.addrs(doffs)], [pe], 0, wide=bb.MxWide.F16) == [bb.ErrorCode.CHECKSUM_MISMATCH]
        assert _counter(cl, "get_placement_refresh_total") == ref + 1
