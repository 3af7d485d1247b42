"""MXFP8 device calls with fp16 and fp32 tensors (`wide=`) on CPU: the HostLoopbackTransport stands in for the GPU fabric
and runs the CPU codec with the call's wide type, so every client rule stated in element bytes -- the virtual-base
alignment, the row-gap rule, replica fail-over -- runs in the CPU suite.  Every result must equal the CPU reference,
and no byte outside a window or a row set may be written."""
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


def _values(rng, n, w):
    """n elements of type w: normal samples over many binades, a few specials."""
    v = (rng.standard_normal(n) * np.exp2(rng.integers(-12, 12, n))).astype(np.float32)
    v[::97] = np.nan
    v[5::211] = np.inf
    v[7::331] = 0.0
    return v.astype(NP[w]) if w != "bf16" else (v.view(np.uint32) >> 16).astype(np.uint16)


def _ref(bb, x, w, out="same"):
    """CPU reference: unpack(pack(x)) as raw bytes of type `out` (default: x's type)."""
    out = w if out == "same" else out
    packed = bb.mxfp8_pack_ref(x, mxw(bb, w))
    return np.frombuffer(bb.mxfp8_unpack_ref(packed, x.size, mxw(bb, out)), dtype=np.uint8)


class Buf:
    """A guard-filled host buffer with a 16-byte aligned region at `at` (+ skew bytes)."""

    def __init__(self, nbytes, skew=0):
        self.raw = np.full(nbytes + 256, GUARD, dtype=np.uint8)
        self.at = (-self.raw.ctypes.data) % 16 + 64 + skew
        self.ptr = self.raw.ctypes.data + self.at

    def expect(self, placed):
        """The whole buffer as it must be: guard everywhere except placed = {byte offset in the region: bytes}."""
        want = np.full_like(self.raw, GUARD)
        for off, b in placed.items():
            want[self.at + off:self.at + off + len(b)] = b
        return want


def _rows_bytes(ref, b, offset, width, pitch, rows):
    e = ref.reshape(-1, b)
    return np.concatenate([e[offset + r * pitch:offset + r * pitch + width].reshape(-1) for r in range(rows)])


def test_six_calls_match_reference_and_keep_guards(bb):
    """All six fp8 calls, for fp16 and fp32, with 2 copies: results equal the CPU reference, guards stay."""
    rng = np.random.default_rng(7)
    with LocalCluster(cluster_id="fp8wide", n_workers=2, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        for w in ("f16", "f32"):
            b, wd = SIZE[w], mxw(bb, w)
            per = 16 // b
            n = 96 * 22 * per  # whole blocks, whole rows of 3 * per and 4 * per, more than a tile
            x = _values(rng, n, w)
            ref = _ref(bb, x, w)
            assert cl.batch_put_device_fp8([f"{w}/a"], [x.ctypes.data], [n], _cfg(bb, 2), 0, wide=wd) == [bb.ErrorCode.OK]
            # strided put: rows of 3 * per elements every 5 * per, read from a buffer whose gaps hold NaN
            rows, width, pitch = n // (3 * per), 3 * per, 5 * per
            src = np.full(rows * pitch, np.nan, dtype=NP[w])
            src.reshape(rows, pitch)[:, :width] = x.reshape(rows, width)
            assert cl.batch_put_device_fp8_strided([f"{w}/s"], [src.ctypes.data], [width], [pitch], [rows], _cfg(bb, 1), 0,
                                                   wide=wd) == [bb.ErrorCode.OK]
            for key in (f"{w}/a", f"{w}/s"):
                # whole
                out = Buf(n * b)
                assert cl.batch_get_device_fp8([key], [out.ptr], [n], 0, wide=wd) == [bb.ErrorCode.OK]
                assert np.array_equal(out.raw, out.expect({0: ref})), (w, key)
                # range: starts mid-block; its virtual base ptr - b * lo is aligned
                lo, cnt = 3 * per + per, n // 2 + 5 * per
                out = Buf(cnt * b, skew=(lo * b) % 16)
                assert cl.batch_get_device_fp8_range([key], [out.ptr], [n], [lo], [cnt], 0, wide=wd) == [bb.ErrorCode.OK]
                assert np.array_equal(out.raw, out.expect({0: ref[lo * b:(lo + cnt) * b]})), (w, key)
                # strided get: rows of 2 * per every 6 * per from element per
                off, gw, gp, gr = per, 2 * per, 6 * per, n // (6 * per) - 1
                out = Buf(gw * gr * b, skew=(off * b) % 16)
                assert cl.batch_get_device_fp8_strided([key], [out.ptr], [n], [off], [gw], [gp], [gr], 0, wide=wd) == [bb.ErrorCode.OK]
                assert np.array_equal(out.raw, out.expect({0: _rows_bytes(ref, b, off, gw, gp, gr)})), (w, key)
                # scatter: rows of 4 * per every 7 * per
                sw, sp = 4 * per, 7 * per
                sr = n // sw
                out = Buf(sr * sp * b)
                assert cl.batch_get_device_fp8_scatter([key], [out.ptr], [n], [sw], [sp], [sr], 0, wide=wd) == [bb.ErrorCode.OK]
                placed = {r * sp * b: ref[r * sw * b:(r + 1) * sw * b] for r in range(sr)}
                assert np.array_equal(out.raw, out.expect(placed)), (w, key)


def test_any_packed_object_reads_into_any_wide_type(bb):
    """An fp32-packed object read as bf16 and fp16 equals the reference unpack to that type; the bytes metrics count
    wide bytes."""
    rng = np.random.default_rng(8)
    with LocalCluster(cluster_id="fp8cross", n_workers=1, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        n = T + 64
        x = _values(rng, n, "f32")
        assert cl.batch_put_device_fp8(["x"], [x.ctypes.data], [n], _cfg(bb, 1), 0, wide=bb.MxWide.F32) == [bb.ErrorCode.OK]
        for out_w in ("bf16", "f16", "f32"):
            out = Buf(n * SIZE[out_w])
            assert cl.batch_get_device_fp8(["x"], [out.ptr], [n], 0, wide=mxw(bb, out_w)) == [bb.ErrorCode.OK]
            assert np.array_equal(out.raw, out.expect({0: _ref(bb, x, "f32", out_w)})), out_w
        before = _counter(cl, "device_get_fp8_range_bytes_total")
        out = Buf(64 * 4)
        assert cl.batch_get_device_fp8_range(["x"], [out.ptr], [n], [0], [64], 0, wide=bb.MxWide.F32) == [bb.ErrorCode.OK]
        assert _counter(cl, "device_get_fp8_range_bytes_total") == before + 64 * 4


def test_fail_over_keeps_guards(bb):
    """With one copy corrupt, each get fails over to the other and writes nothing outside its window or rows."""
    rng = np.random.default_rng(9)
    with LocalCluster(cluster_id="fp8widefo", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        pools = {p.id: p for p in cl.keystone().get_memory_pools()}

        def flip(sh, pos):
            wk = [wk for wk in c.workers if wk.backend(sh.pool_id) is not None][0]
            off = sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr + pos
            be = wk.backend(sh.pool_id)
            be.write(off, bytes([be.read(off, 1)[0] ^ 0xFF]))

        for w in ("f16", "f32"):
            b, wd, per = SIZE[w], mxw(bb, w), 16 // SIZE[w]
            n = T + 32 * per
            x = _values(rng, n, w)
            ref = _ref(bb, x, w)
            assert cl.batch_put_device_fp8([w], [x.ctypes.data], [n], _cfg(bb, 2), 0, wide=wd) == [bb.ErrorCode.OK]
            for sh in [cp.shards[0] for cp in cl.get_workers(w)]:
                flip(sh, 100)
                fo = _counter(cl, "replica_failover_total")
                outs = [Buf(n * b), Buf(per * 4 * b), Buf(n // (4 * per) * 8 * per * b)]
                ok = bb.ErrorCode.OK
                assert cl.batch_get_device_fp8([w], [outs[0].ptr], [n], 0, wide=wd) == [ok]
                assert cl.batch_get_device_fp8_range([w], [outs[1].ptr], [n], [0], [4 * per], 0, wide=wd) == [ok]
                assert cl.batch_get_device_fp8_scatter([w], [outs[2].ptr], [n], [4 * per], [8 * per], [n // (4 * per)], 0, wide=wd) == [ok]
                assert np.array_equal(outs[0].raw, outs[0].expect({0: ref}))
                assert np.array_equal(outs[1].raw, outs[1].expect({0: ref[:4 * per * b]}))
                rs, rw = 8 * per * b, 4 * per * b
                assert np.array_equal(outs[2].raw, outs[2].expect({r * rs: ref[r * rw:(r + 1) * rw] for r in range(n // (4 * per))}))
                assert _counter(cl, "replica_failover_total") >= fo
                flip(sh, 100)  # restore


def test_alignment_rules_in_element_bytes(bb):
    """fp32: a row gap of 4 elements is fusable where bf16 refuses it (NOT_IMPLEMENTED); a gap of 2 elements is refused;
    a range whose virtual base ptr - 4 * lo is not 16-byte aligned is refused.  Each refused item fails alone."""
    rng = np.random.default_rng(10)
    NI, OK = bb.ErrorCode.NOT_IMPLEMENTED, bb.ErrorCode.OK
    with LocalCluster(cluster_id="fp8widealign", n_workers=1, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        n = T
        xb = _values(rng, n, "bf16")
        assert cl.batch_put_device_fp8(["bf16"], [xb.ctypes.data], [n], _cfg(bb, 1), 0) == [OK]
        x32 = _values(rng, n, "f32")
        ref = _ref(bb, x32, "f32")
        assert cl.batch_put_device_fp8(["f32"], [x32.ctypes.data], [n], _cfg(bb, 1), 0, wide=bb.MxWide.F32) == [OK]
        # scatter: width 28, pitch 32 (gap 4) and pitch 30 (gap 2)
        for w, pitch, want in (("f32", 32, OK), ("bf16", 32, NI), ("f32", 30, NI)):
            out = Buf(n // 28 * pitch * 4 + 256)
            rows = n // 28
            m = rows * 28
            got = cl.batch_get_device_fp8_scatter([w], [out.ptr], [n], [28], [pitch], [rows], 0, wide=mxw(bb, w))
            assert got == [bb.ErrorCode.INVALID_ARGUMENT if m != n else want], (w, pitch)
        out = Buf(n // 32 * 36 * 4)
        assert cl.batch_get_device_fp8_scatter(["f32"], [out.ptr], [n], [32], [36], [n // 32], 0, wide=bb.MxWide.F32) == [OK]
        assert np.array_equal(out.raw, out.expect({r * 36 * 4: ref[r * 128:(r + 1) * 128] for r in range(n // 32)}))
        out = Buf(n // 32 * 40 * 2)
        assert cl.batch_get_device_fp8_scatter(["bf16"], [out.ptr], [n], [32], [36], [n // 32], 0) == [NI]
        # strided get: width 12, pitch 16 (gap 4) from element 4
        for w, want in (("f32", OK), ("bf16", NI)):
            b = SIZE[w]
            out = Buf(12 * 100 * b, skew=(4 * b) % 16)
            got = cl.batch_get_device_fp8_strided([w], [out.ptr], [n], [4], [12], [16], [100], 0, wide=mxw(bb, w))
            assert got == [want], w
            if w == "f32":
                assert np.array_equal(out.raw, out.expect({0: _rows_bytes(ref, 4, 4, 12, 16, 100)}))
            else:
                assert np.array_equal(out.raw, out.expect({}))
        # strided put: the same rows as a source
        src = np.zeros(16 * 100 * 2, dtype=np.float32)
        for w, want in (("f32", OK), ("bf16", NI)):
            got = cl.batch_put_device_fp8_strided([f"p/{w}"], [src.ctypes.data], [16], [20], [64], _cfg(bb, 1), 0, wide=mxw(bb, w))
            assert got == [want], w
        got = cl.batch_put_device_fp8_strided(["p/odd"], [src.ctypes.data], [16], [18], [64], _cfg(bb, 1), 0, wide=bb.MxWide.F32)
        assert got == [NI]
        # range: the virtual base ptr - 4 * lo must be 16-byte aligned; lo = 1 at an aligned pointer is refused, and the
        # rest of the batch still goes
        out = Buf(64 * 4)
        got = cl.batch_get_device_fp8_range(["f32", "f32"], [out.ptr, out.ptr + 4], [n, n], [1, 1], [8, 8], 0, wide=bb.MxWide.F32)
        assert got == [NI, OK]
        assert np.array_equal(out.raw, out.expect({4: ref[4:36]}))
