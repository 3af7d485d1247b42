"""Segment-list puts and gets of MXFP8-packed tensors (batch_put_device_fp8_segments, batch_get_device_fp8_segments) on
CPU: the SourceSegments rule in element units against an independent numpy model, and both client calls through the
HostLoopbackTransport, which stands in for the GPU fabric and runs the CPU codec, so the client's rules -- the table in
wide bytes, co-alignment, whole MX blocks, the refusals, replica fan-out, fail-over and the placement refresh -- run in
the CPU suite.  Segment addresses here are host addresses: the loopback's "device pointers" are host pointers."""
import json

import numpy as np
import pytest

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


def _unpacked(bb, blob, w, n, out_w=None):
    """The wide bytes a get of type out_w returns for a packed put of blob (n elements of type w)."""
    out_w = out_w or w
    return np.frombuffer(bb.mxfp8_unpack_ref(bb.mxfp8_pack_ref(blob.view(NP[w]), mxw(bb, w)), n, mxw(bb, out_w)), np.uint8)


# ---------------------------------------------------------------- the rule in element units against a numpy model
def model_bytes(segs, b):
    """Per wide byte of the object: its address, or -1 inside a null segment, for (address, elements) segments."""
    addr = []
    for a, n in segs:
        addr += [a + i if a else -1 for i in range(b * n)]
    return np.array(addr, dtype=np.int64)


def model_runs(addr, lo, hi, b):
    """Maximal runs of wide bytes [lo, hi) whose addresses follow one another, null bytes in none, as (x, addr, n) in
    elements from lo."""
    out, x = [], lo
    while x < hi:
        if addr[x] < 0:
            x += 1
            continue
        y = x + 1
        while y < hi and addr[y] >= 0 and addr[y] == addr[y - 1] + 1:
            y += 1
        out.append(((x - lo) // b, int(addr[x]), (y - x) // b))
        x = y
    return out


def model_coaligned(addr, lo, hi):
    """Every non-null wide byte x of [lo, hi) lives at an address congruent to x - lo mod 16."""
    x = np.arange(lo, hi)
    a = addr[lo:hi]
    return bool(np.all((a < 0) | ((a - (x - lo)) % 16 == 0)))


def test_element_rule_and_to_wide_bytes_match_the_numpy_model(bb):
    rng = np.random.default_rng(21)
    for trial in range(200):
        b = int(rng.choice([2, 4]))
        segs, base, off = [], int(rng.integers(1, 1 << 30)) * 16, 0
        for _ in range(int(rng.integers(1, 30))):
            n = int(rng.choice([0, 1, 3, 7, 23, 32, 33, 500, T // b + 5]))
            if rng.random() < 0.1:
                a = 0
            elif segs and segs[-1][0] and rng.random() < 0.3:
                a = segs[-1][0] + b * segs[-1][1]  # adjacent in memory: one run
            else:
                base += int(rng.integers(1, 1 << 16)) * 16
                a = base + ((b * off) % 16 if trial % 2 == 0 else int(rng.integers(0, 8)) * 2)
            segs.append((a, n))
            off += n
        ec, t, size = bb.SourceSegments.from_segments(segs, elem_bytes=b)
        assert ec == bb.ErrorCode.OK and size == off
        kept = [(a, n) for a, n in segs if n]
        if not kept:
            assert not t.segmented()
            continue
        assert t.unit == b
        starts = np.concatenate([[0], np.cumsum([n for _, n in kept])]).astype(int).tolist()
        assert t.entries == [(b * starts[k], kept[k][0]) for k in range(len(kept))] + [(b * size, 0)]  # the table is in bytes
        addr = model_bytes(kept, b)
        assert t.to_wide_bytes(6 - b) is None and t.to_wide_bytes(1) is None
        w = t.to_wide_bytes(b)
        assert w.unit == 1 and w.entries == t.entries and w.phase == 0  # the same table, unit 1
        cuts = sorted(set([0, size] + starts + [int(c) for c in rng.integers(0, size + 1, 5)]))
        for lo, hi in zip(cuts, cuts[1:] + [size]):
            r, n = t.rebase(lo), hi - lo
            assert r.phase == b * lo and r.unit == b and r.valid(n) and not r.valid(size - lo + 1)
            assert r.runs(n) == model_runs(addr, b * lo, b * hi, b)
            assert r.has_null(n) == bool(np.any(addr[b * lo:b * hi] < 0))
            assert r.coaligned(n) == model_coaligned(addr, b * lo, b * hi)
            assert t.fused_get_aligned(lo, n) == model_coaligned(addr, b * lo, b * hi)
            rw = r.to_wide_bytes(b)  # wide bytes: the byte rule of the same table
            assert rw.phase == r.phase and rw.segments_for(b * n) == r.segments_for(n) and rw.coaligned(b * n) == r.coaligned(n)
            assert [(x * b, a, c * b) for x, a, c in r.runs(n)] == rw.runs(b * n)
    # a segment's or the total's wide bytes overflow
    assert bb.SourceSegments.from_segments([(16, 1 << 63)], elem_bytes=2)[0] == bb.ErrorCode.VALUE_OUT_OF_RANGE
    assert bb.SourceSegments.from_segments([(16, 1 << 61), (32, 1 << 61)], elem_bytes=4)[0] == bb.ErrorCode.VALUE_OUT_OF_RANGE
    assert bb.SourceSegments.from_segments([(16, 1 << 61), (32, 1 << 61)], elem_bytes=2)[0] == bb.ErrorCode.OK
    with pytest.raises(ValueError):
        bb.SourceSegments.from_segments([(16, 4)], elem_bytes=0)


# ---------------------------------------------------------------- client calls through the loopback transport
class Arena:
    """One guard-filled host buffer that segments are carved from, each at an address congruent to b times its element
    offset mod 16 (plus a skew in bytes), with guard bytes between them."""

    def __init__(self, nbytes):
        self.raw = np.full(nbytes, GUARD, dtype=np.uint8)
        self.base = self.raw.ctypes.data
        self.o = (-self.base) % 16 + 64

    def segments(self, lens, b, skew=0):
        offs, start = [], 0
        for n in lens:
            self.o = (self.o + 15) // 16 * 16 + 32
            offs.append(self.o + (b * start + skew) % 16)
            self.o = offs[-1] + b * n
            start += n
        assert self.o + 64 < len(self.raw)
        return offs

    def pairs(self, offs, lens, null=()):
        return [(0 if k in null else self.base + o, n) for k, (o, n) in enumerate(zip(offs, lens))]

    def fill(self, offs, lens, b, blob, null=()):
        x = 0
        for k, (o, n) in enumerate(zip(offs, lens)):
            if k not in null:
                self.raw[o:o + b * n] = blob[x:x + b * n]
            x += b * n

    def expect(self, offs, lens, b, blob, null=()):
        """The whole buffer as it must be: guard everywhere except blob cut into the non-null segments."""
        want = np.full_like(self.raw, GUARD)
        raw, self.raw = self.raw, want
        self.fill(offs, lens, b, blob, null)
        self.raw = raw
        return want


# element lengths: MX blocks straddle segments, zero-length and one-element segments, one segment over many tiles
def _lens(rng):
    lens = [int(rng.choice([0, 1, 5, 23, 32, 100, 4096, T + 7, 3 * T])) for _ in range(int(rng.integers(1, 14)))]
    lens.append(-sum(lens) % 32 + 32)  # a whole number of MX blocks
    return lens


def test_put_equals_a_packed_put_of_the_concatenation(bb):
    """Co-aligned segments with guard gaps, for bf16, fp16 and fp32: the stored bytes are the reference packing of the
    concatenation, the digests those of batch_put_device_fp8 of it, and both objects read back through plain fp8 gets
    and segment gets into differently cut segments with null ones."""
    rng = np.random.default_rng(22)
    with LocalCluster(cluster_id="fp8sg", n_workers=2, pool_bytes=96 * MiB) as c:
        cl = make_client(bb, c)
        n0 = _counter(cl, "device_put_fp8_segments_total")
        for w in ("bf16", "f16", "f32"):
            b, wd = SIZE[w], mxw(bb, w)
            shapes = [_lens(rng) for _ in range(4)]
            ar = Arena(sum(b * sum(ls) + 64 * len(ls) for ls in shapes) + MiB)
            keys, lists, blobs = [], [], []
            for j, lens in enumerate(shapes):
                offs = ar.segments(lens, b)
                blob = _values(rng, sum(lens), w)
                ar.fill(offs, lens, b, blob)
                keys.append(f"{w}/{j}"), lists.append(ar.pairs(offs, lens)), blobs.append(blob)
            before = ar.raw.copy()
            assert cl.batch_put_device_fp8_segments(keys, lists, _cfg(bb, 2), 0, wide=wd) == [bb.ErrorCode.OK] * 4
            assert np.array_equal(ar.raw, before)  # a put reads only
            for (ec, stored), blob, key in zip(cl.batch_get(keys), blobs, keys):
                assert ec == bb.ErrorCode.OK and bytes(stored) == bb.mxfp8_pack_ref(blob.view(NP[w]), wd), key
                assert len(cl.get_workers(key)) == 2
            refs = [k + "/ref" for k in keys]
            assert cl.batch_put_device_fp8(refs, [x.ctypes.data for x in blobs], [x.size // b for x in blobs], _cfg(bb, 2), 0,
                                           wide=wd) == [bb.ErrorCode.OK] * 4
            for k, r in zip(keys, refs):
                assert _sums(cl, k) == _sums(cl, r), k
            for j, lens in enumerate(shapes):
                n = sum(lens)
                want = _unpacked(bb, blobs[j], w, n)
                out = np.zeros(b * n, np.uint8)
                assert cl.batch_get_device_fp8([keys[j]], [out.ctypes.data], [n], 0, wide=wd) == [bb.ErrorCode.OK]
                assert np.array_equal(out, want), (w, j)
                # the plain object into segments cut elsewhere, some null
                cuts = sorted(set(int(x) for x in rng.integers(0, n + 1, 6)) | {0, n})
                lens2 = [y - x for x, y in zip(cuts, cuts[1:])]
                null = {k for k in range(len(lens2)) if rng.random() < 0.3}
                dst = Arena(b * n + 64 * len(lens2) + 4096)
                doffs = dst.segments(lens2, b)
                ecs, sizes = cl.batch_get_device_fp8_segments([refs[j]], [dst.pairs(doffs, lens2, null)], 0, wide=wd)
                assert ecs == [bb.ErrorCode.OK] and sizes == [n]
                assert np.array_equal(dst.raw, dst.expect(doffs, lens2, b, want, null)), (w, j)
        assert _counter(cl, "device_put_fp8_segments_total") == n0 + 12
        assert _counter(cl, "device_get_fp8_segments_total") == 12


def test_any_packed_object_reads_into_segments_of_any_wide_type(bb):
    """A bf16 object put from segments reads into fp32 segments, and an fp32 plain object into bf16 segments."""
    rng = np.random.default_rng(23)
    with LocalCluster(cluster_id="fp8sgx", n_workers=1, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        lens = [5, 300, 27, 4096, 116]  # 4544 elements = 142 blocks
        src = Arena(4 * sum(lens) + 4096)
        offs = src.segments(lens, 2)
        blob = _values(rng, sum(lens), "bf16")
        src.fill(offs, lens, 2, blob)
        assert cl.batch_put_device_fp8_segments(["x"], [src.pairs(offs, lens)], _cfg(bb, 1), 0) == [bb.ErrorCode.OK]
        dst = Arena(4 * sum(lens) + 4096)
        doffs = dst.segments(lens, 4)
        ecs, _ = cl.batch_get_device_fp8_segments(["x"], [dst.pairs(doffs, lens)], 0, wide=bb.MxWide.F32)
        assert ecs == [bb.ErrorCode.OK]
        assert np.array_equal(dst.raw, dst.expect(doffs, lens, 4, _unpacked(bb, blob, "bf16", sum(lens), "f32")))
        f32 = _values(rng, sum(lens), "f32")
        assert cl.batch_put_device_fp8(["y"], [f32.ctypes.data], [sum(lens)], _cfg(bb, 1), 0, wide=bb.MxWide.F32) == [bb.ErrorCode.OK]
        dst = Arena(2 * sum(lens) + 4096)
        doffs = dst.segments(lens, 2)
        ecs, _ = cl.batch_get_device_fp8_segments(["y"], [dst.pairs(doffs, lens)], 0, wide=bb.MxWide.BF16)
        assert ecs == [bb.ErrorCode.OK]
        assert np.array_equal(dst.raw, dst.expect(doffs, lens, 2, _unpacked(bb, f32, "f32", sum(lens), "bf16")))


def test_refusals_fail_alone(bb):
    """Every refusal gives its per-object code before anything is allocated (puts) or read, while the rest of the batch
    succeeds; nothing is written outside the accepted items' segments."""
    rng = np.random.default_rng(24)
    E = bb.ErrorCode
    with LocalCluster(cluster_id="fp8sgr", n_workers=1, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        ar = Arena(2 * MiB)
        lens = [100, 28, 4000]  # 4128 elements = 129 blocks
        good = ar.segments(lens, 2)
        blob = _values(rng, sum(lens), "bf16")
        ar.fill(good, lens, 2, blob)
        skewed = ar.segments(lens, 2, skew=2)  # one element off its co-aligned address
        keys = ["ok", "null", "part", "empty", "ovf", "skew", "ok2"]
        lists = [ar.pairs(good, lens), ar.pairs(good, lens, {1}), ar.pairs(good, [100, 28, 3990]), [], [(ar.base, 1 << 63)],
                 ar.pairs(skewed, lens), ar.pairs(good, lens)]
        ecs = cl.batch_put_device_fp8_segments(keys, lists, _cfg(bb, 1), 0)
        assert ecs == [E.OK, E.INVALID_ARGUMENT, E.INVALID_ARGUMENT, E.INVALID_ARGUMENT, E.VALUE_OUT_OF_RANGE, E.NOT_IMPLEMENTED, E.OK]
        for k in ("null", "part", "empty", "ovf", "skew"):
            assert not cl.object_exists(k), k
        # gets: size mismatch (one element short of the object, and one block more), not whole blocks, nothing,
        # misaligned, missing key, null segments, OK
        dst = Arena(2 * MiB)
        d = dst.segments(lens, 2)
        more = dst.segments(lens + [32], 2)
        dskew = dst.segments(lens, 2, skew=6)
        snapshot = dst.raw.copy()
        ecs, sizes = cl.batch_get_device_fp8_segments(
            ["ok", "ok", "ok", "ok", "ok", "nope", "ok", "ok2"],
            [dst.pairs(d, [100, 28, 3968]) + [(0, 31)], dst.pairs(more, lens + [32]), dst.pairs(d, [100, 28, 3990]), [],
             dst.pairs(dskew, lens), dst.pairs(d, lens), [(0, 100), (0, 28), (0, 4000)], dst.pairs(d, lens, {0})], 0)
        assert ecs == [E.INVALID_ARGUMENT, E.INVALID_ARGUMENT, E.INVALID_ARGUMENT, E.INVALID_ARGUMENT, E.NOT_IMPLEMENTED,
                       E.OBJECT_NOT_FOUND, E.OK, E.OK], ecs
        assert sizes == [0] * 6 + [4128, 4128]
        dst.raw, got = snapshot, dst.raw  # only ok2's non-null segments are written
        dst.fill(d, lens, 2, _unpacked(bb, blob, "bf16", sum(lens)), {0})
        assert np.array_equal(got, snapshot)
        # arity
        assert cl.batch_put_device_fp8_segments(["a", "b"], [[]], _cfg(bb, 1), 0) == [E.INVALID_PARAMETERS] * 2
        assert cl.batch_get_device_fp8_segments(["a", "b"], [[]], 0)[0] == [E.INVALID_PARAMETERS] * 2


def test_fail_over_and_refresh(bb):
    """A corrupt copy fails the segment get over to the next replica, segments right and guards untouched; with every
    copy corrupt the object is re-read once (placement refresh) and the answer is CHECKSUM_MISMATCH."""
    rng = np.random.default_rng(25)
    with LocalCluster(cluster_id="fp8sgf", n_workers=3, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        pools = {p.id: p for p in cl.keystone().get_memory_pools()}

        def flip(sh, pos):
            wk = [wk for wk in c.workers if wk.backend(sh.pool_id) is not None][0]
            off = sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr + pos
            be = wk.backend(sh.pool_id)
            be.write(off, bytes([be.read(off, 1)[0] ^ 0xFF]))

        lens = [int(x) for x in rng.integers(1, 3000, 40)]
        lens.append(-sum(lens) % 32 + 32)
        n = sum(lens)
        src = Arena(2 * n + 64 * len(lens) + 4096)
        offs = src.segments(lens, 2)
        blob = _values(rng, n, "f16")
        src.fill(offs, lens, 2, blob)
        assert cl.batch_put_device_fp8_segments(["f"], [src.pairs(offs, lens)], _cfg(bb, 3), 0, wide=bb.MxWide.F16) == [bb.ErrorCode.OK]
        want = _unpacked(bb, blob, "f16", n)
        copies = cl.get_workers("f")
        assert len(copies) == 3
        fo = _counter(cl, "replica_failover_total")
        for cp in copies:
            flip(cp.shards[0], 4321)
            dst = Arena(2 * n + 64 * len(lens) + 4096)
            doffs = dst.segments(lens, 2)
            ecs, _ = cl.batch_get_device_fp8_segments(["f"], [dst.pairs(doffs, lens)], 0, wide=bb.MxWide.F16)
            assert ecs == [bb.ErrorCode.OK]
            assert np.array_equal(dst.raw, dst.expect(doffs, lens, 2, want))
            flip(cp.shards[0], 4321)
        assert _counter(cl, "replica_failover_total") > fo
        for cp in copies:
            flip(cp.shards[0], 7)
        ref = _counter(cl, "get_placement_refresh_total")
        dst = Arena(2 * n + 64 * len(lens) + 4096)
        ecs, _ = cl.batch_get_device_fp8_segments(["f"], [dst.pairs(dst.segments(lens, 2), lens)], 0, wide=bb.MxWide.F16)
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH]
        assert _counter(cl, "get_placement_refresh_total") == ref + 1


# ---------------------------------------------------------------- TensorStore checks that need no GPU
def test_tensor_store_packed_bundle_checks_before_any_transfer(monkeypatch):
    torch = pytest.importorskip("torch")
    from blackbird_b200 import _bb
    from blackbird_b200.ops import TensorStore

    meta = {"bundle": "dict", "entries": [{"name": "w", "dtype": "bfloat16", "shape": [4], "offset": 0, "bytes": 8}], "total": 64,
            "packed": "mxfp8", "dtype": "bfloat16", "numel": 32}

    class MetasOnly:
        """Answers the `#meta` reads and nothing else: any transfer fails the test."""

        def batch_get(self, keys):
            assert all(k.endswith("#meta") for k in keys)
            return [(_bb.ErrorCode.OK, json.dumps(meta).encode()) for _ in keys]

        def __getattr__(self, name):
            raise AssertionError(f"client.{name} called")

    ts = TensorStore.__new__(TensorStore)
    ts.client, ts.config = MetasOnly(), None
    with pytest.raises(TypeError, match="one dtype"):
        ts.batch_put_bundles(["k"], [{"a": torch.zeros(4, dtype=torch.bfloat16), "b": torch.zeros(4, dtype=torch.float16)}], pack_fp8=True)
    with pytest.raises(TypeError, match="one dtype"):
        ts.put_bundle("k", [torch.zeros(4, dtype=torch.int32)], pack_fp8=True)
    with pytest.raises(TypeError, match="one dtype"):
        ts.put_bundle("k", [torch.zeros(4, dtype=torch.float64)], None, True)
    with pytest.raises(ValueError, match="CUDA"):
        ts.put_bundle("k", {"w": torch.zeros(4, dtype=torch.float32)}, pack_fp8=True)  # a CPU tensor
    with pytest.raises(ValueError, match="at least one element"):
        ts.put_bundle("k", {}, pack_fp8=True)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)  # the out checks name the current device
    with pytest.raises(TypeError, match="out is torch.float16"):
        ts.get_bundle_into("k", {"w": torch.zeros(4, dtype=torch.float16)})
    with pytest.raises(ValueError, match="shape"):
        ts.get_bundle_into("k", {"w": torch.zeros(5, dtype=torch.bfloat16)})
    with pytest.raises(KeyError):
        ts.get_bundle_into("k", {"v": torch.zeros(4, dtype=torch.bfloat16)})
    with pytest.raises(ValueError, match="CUDA"):
        ts.get_bundle_into("k", {"w": torch.zeros(4, dtype=torch.bfloat16)})
