"""Slice gets into existing tensors on CPU: the WindowRows rule (common/store_window.h) against an independent numpy model,
and batch_get_device_strided_scatter / batch_get_device_fp8_strided_scatter through the HostLoopbackTransport, which
follows the rule as the fused kernels do: striped objects, host staging, refusals and the TensorStore checks that come
before any transfer."""
import os
import random

import numpy as np
import pytest

from blackbird_b200.parallel import LocalCluster

MiB = 1 << 20
GUARD = 0xA5


# ---------------------------------------------------------------------------------------------------- the numpy model


def model_pairs(offset, width, pitch, rows, dw, dp, dph):
    """(object index, destination index) of every stored unit: the window's rows land densely as result index p, which
    lands at ((p + dph) // dw) * dp + (p + dph) % dw."""
    r = np.arange(rows, dtype=np.int64)[:, None]
    c = np.arange(width, dtype=np.int64)[None, :]
    x = (offset + r * pitch + c).ravel()
    p = (r * width + c).ravel()
    q = p + dph
    return x, (q // dw) * dp + q % dw


def runs_pairs(runs):
    xs = [np.arange(x, x + n, dtype=np.int64) for x, _, n in runs]
    ats = [np.arange(a, a + n, dtype=np.int64) for _, a, n in runs]
    if not xs:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(xs), np.concatenate(ats)


def random_shape(rng, size):
    width = rng.randint(1, 300)
    pitch = width + rng.choice([0, rng.randint(1, 64), 16 * rng.randint(1, 8)])
    rows = rng.randint(1, 12)
    if (rows - 1) * pitch + width > size:
        rows = max(1, (size - width) // pitch + 1) if width <= size else 0
    offset = rng.randint(0, max(0, size - ((rows - 1) * pitch + width))) if rows else 0
    dw = rng.randint(1, 200)
    dp = dw + rng.choice([0, rng.randint(1, 40), 16 * rng.randint(1, 4)])
    dph = rng.randint(0, dw - 1)
    return offset, width, pitch, rows, dw, dp, dph


def test_rule_runs_match_the_model_at_every_phase(bb):
    rng = random.Random(7)
    n = 0
    for _ in range(600):
        size = rng.randint(1, 5000)
        offset, width, pitch, rows, dw, dp, dph = random_shape(rng, size)
        if rows == 0:
            continue
        ec, w = bb.WindowRows.from_rows(offset, width, pitch, rows, size, bb.SourceRows(dp, dw, dph))
        assert ec == bb.ErrorCode.OK
        assert w.valid(size)
        x, d = runs_pairs(w.runs(size))
        mx, md = model_pairs(offset, width, pitch, rows, dw, dp, dph)
        assert np.array_equal(x, mx) and np.array_equal(d, md), (offset, width, pitch, rows, dw, dp, dph)
        for k in range(0, len(mx), max(1, len(mx) // 7)):
            assert w.at(w.index(int(mx[k]))) == md[k]
        # every run lies inside one destination row
        for _, at, k in w.runs(size):
            q = at % dp if dp != dw else None
            if q is not None:
                assert q + k <= dw
        n += 1
    assert n > 500


def test_rows_without_a_pattern_are_the_windows_own_get(bb):
    ec, w = bb.WindowRows.from_rows(100, 30, 50, 4, 1000, bb.SourceRows())
    assert ec == bb.ErrorCode.OK
    x, d = runs_pairs(w.runs(1000))
    mx, _ = model_pairs(100, 30, 50, 4, 1, 1, 0)
    assert np.array_equal(x, mx) and np.array_equal(d, np.arange(120))


def brute_coaligned(w, dst, size):
    x, d = runs_pairs(w.runs(size))
    return bool(np.all((dst + d - x) % 16 == 0))


def test_coalignment_verdicts(bb):
    rng = random.Random(11)
    exact = sound = 0
    for _ in range(1500):
        size = rng.randint(1, 4000)
        offset, width, pitch, rows, dw, dp, dph = random_shape(rng, size)
        if rows == 0:
            continue
        # bias the shapes towards congruent ones, so that both verdicts occur
        if rng.random() < 0.6:
            pitch = width + 16 * rng.randint(0, 3) if rows > 1 else pitch
            dp = dw + 16 * rng.randint(0, 3)
            if (rows - 1) * pitch + width > size:
                continue
        ec, w = bb.WindowRows.from_rows(offset, width, pitch, rows, size, bb.SourceRows(dp, dw, dph))
        dst = rng.randint(0, 64) + 4096
        if rng.random() < 0.5:  # the first stored byte congruent
            dst += (offset - w.at(0) - dst) % 16
        got, want = w.coaligned(dst, size), brute_coaligned(w, dst, size)
        assert not got or want, (offset, width, pitch, rows, dw, dp, dph, dst)  # never passes a misaligned shape
        gaps16 = (pitch - width) % 16 == 0 and (dp - dw) % 16 == 0
        if gaps16:
            assert got == want
            exact += 1
        sound += got
    assert exact > 300 and sound > 100
    # heads and tails under 16 bytes on both sides: rows of 5 bytes every 21 into rows of 7 every 23
    ec, w = bb.WindowRows.from_rows(3, 5, 21, 30, 1000, bb.SourceRows(23, 7, 2))
    assert not w.coaligned(4096, 1000)
    ec, w = bb.WindowRows.from_rows(3, 5, 21, 30, 1000, bb.SourceRows(39, 7, 2))
    assert w.coaligned(4096 + 1, 1000) == brute_coaligned(w, 4096 + 1, 1000)


def test_shard_rebasing_follows_the_first_stored_unit(bb):
    rng = random.Random(3)
    for _ in range(300):
        size = rng.randint(50, 6000)
        offset, width, pitch, rows, dw, dp, dph = random_shape(rng, size)
        if rows == 0:
            continue
        ec, w = bb.WindowRows.from_rows(offset, width, pitch, rows, size, bb.SourceRows(dp, dw, dph))
        mx, md = model_pairs(offset, width, pitch, rows, dw, dp, dph)
        cuts = sorted(set([0, size] + [rng.randint(1, size - 1) for _ in range(rng.randint(0, 4))]))
        got_x, got_d = [], []
        for a, b in zip(cuts, cuts[1:]):
            lo, hi = w.window[0], w.window[1]
            if not (a < hi and b > lo):  # the client rebases only the shards the window touches
                continue
            r, shift = w.rebase(a, b - a)
            x, d = runs_pairs(r.runs(b - a))
            got_x.append(x + a)
            got_d.append(d + shift)
            # with 16-byte gaps the shard's closed-form verdict is the brute-force one over its own offsets
            if (pitch - width) % 16 == 0 and (dp - dw) % 16 == 0:
                dst = 4096 + rng.randint(0, 15)
                assert r.coaligned(dst + shift, b - a) == brute_coaligned(r, dst + shift, b - a)
        x, d = np.concatenate(got_x), np.concatenate(got_d)
        assert np.array_equal(x, mx) and np.array_equal(d, md), (offset, width, pitch, rows, dw, dp, dph, cuts)


def test_fused_alignment_is_decided_by_the_call(bb):
    # a gap that is not a multiple of 16 on either side refuses every shard, even one that holds a single row
    ec, w = bb.WindowRows.from_rows(0, 64, 72, 10, 1000, bb.SourceRows(128, 64, 0))
    assert not w.fused_get_aligned(4096, 0, 64)
    ec, w = bb.WindowRows.from_rows(0, 64, 80, 10, 1000, bb.SourceRows(72, 64, 0))
    assert not w.fused_get_aligned(4096, 0, 64)
    ec, w = bb.WindowRows.from_rows(16, 64, 80, 10, 1000, bb.SourceRows(96, 64, 0))
    assert all(w.fused_get_aligned(4096 + 16, a, 128) for a in range(0, 1024, 128))  # shards cut at 16-byte multiples
    assert not w.fused_get_aligned(4096 + 8, 0, 1000)
    # a shard the window does not touch never refuses
    assert w.fused_get_aligned(4096 + 3, 900, 100)


def test_wide_bytes_and_kernel_rows(bb):
    rng = random.Random(5)
    for _ in range(300):
        size = rng.randint(10, 3000)
        offset, width, pitch, rows, dw, dp, dph = random_shape(rng, size)
        if rows == 0:
            continue
        ec, w = bb.WindowRows.from_rows(offset, width, pitch, rows, size, bb.SourceRows(dp, dw, dph))
        for b in (2, 4):
            wb = w.to_wide_bytes(b)
            x, d = runs_pairs(wb.runs(b * size))
            mx, md = model_pairs(offset, width, pitch, rows, dw, dp, dph)
            ex = (mx[:, None] * b + np.arange(b)).ravel()
            ed = (md[:, None] * b + np.arange(b)).ravel()
            assert np.array_equal(x, ex) and np.array_equal(d, ed)
        # the kernels count a strided window's index from pattern row 0: q = ((x + phase) // pitch) * width + c
        lo, hi, wp, ww, wph, row = w.window
        kr, shift = w.kernel_rows()
        mx, md = model_pairs(offset, width, pitch, rows, dw, dp, dph)
        for k in range(0, len(mx), max(1, len(mx) // 5)):
            xx = int(mx[k])
            q = ((xx + wph) // wp) * ww + (xx + wph) % wp if wp else xx - lo
            qq = q + kr.phase
            at = (qq // kr.width) * kr.pitch + qq % kr.width
            assert (at + shift) % 2**64 == md[k], (offset, width, pitch, rows, dw, dp, dph)


# ---------------------------------------------------------------------------------------------------- the client


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


def _cfg(bb, replicas, stripes, algo="XXH3"):
    return bb.WorkerConfig(replication_factor=replicas, max_workers_per_copy=stripes, ttl_ms=0, checksum=getattr(bb.ChecksumAlgo, algo),
                           preferred_classes=[bb.StorageClass.RAM_CPU])


def _buffer(n):
    raw = np.full(n + 256, GUARD, dtype=np.uint8)
    return raw, (-raw.ctypes.data) % 64 + 64


def _slice_gets(bb, cl, keys, blobs, specs):
    """One batch_get_device_strided_scatter of specs (offset, width, pitch, rows, dw, dp, skew) into one guard-filled
    buffer; returns (codes, buffer, expected buffer for the OK items)."""
    total = sum(((s[3] * s[1] + s[4]) // s[4] + 1) * s[5] + 128 for s in specs)
    raw, base = _buffer(total)
    dsts, o = [], base
    for s in specs:
        dsts.append(o + s[6])
        o += ((s[3] * s[1] + s[4]) // s[4] + 1) * s[5] + 128
    ecs = cl.batch_get_device_strided_scatter(keys, [raw.ctypes.data + d for d in dsts], [s[0] for s in specs], [s[1] for s in specs],
                                              [s[2] for s in specs], [s[3] for s in specs], [s[4] for s in specs], [s[5] for s in specs], 0)
    want = np.full_like(raw, GUARD)
    for d, b, s, e in zip(dsts, blobs, specs, ecs):
        if e == bb.ErrorCode.OK:
            x, t = model_pairs(s[0], s[1], s[2], s[3], s[4], s[5], 0)
            want[d + t] = b[x]
    return ecs, raw, want


def test_client_slice_gets_over_striped_objects(bb):
    with LocalCluster(cluster_id="slicecpu", n_workers=4, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        size = 2 * MiB + 4321
        blob = np.frombuffer(os.urandom(size), dtype=np.uint8).copy()
        assert cl.batch_put_device(["s"], [blob.ctypes.data], [size], _cfg(bb, 2, 4), 0) == [bb.ErrorCode.OK]
        # (offset, width, pitch, rows, dst width, dst pitch, dst skew): ranges (one row) and strided windows across the
        # stripe cuts, into rows with and without 16-byte gaps, heads and tails under 16 bytes
        specs = [(0, size, size, 1, 4096, 4096 + 512, 0),        # the whole object into rows
                 (5, 100000, 100000, 1, 777, 777 + 33, 3),      # a range, rows of odd width and gap
                 (64, 4096, 8192, 200, 4096, 4096 + 1024, 0),   # a TP column shard into a fused parameter
                 (16, 1024, 4096, 300, 512, 2048, 0),           # window rows wider than destination rows
                 (3, 5, 21, 5000, 7, 23, 1),                    # both sides short and unaligned
                 (100, 48, 16384, 100, 4096, 8192, 0)]          # destination rows wider than the window's
        ecs, raw, want = _slice_gets(bb, cl, ["s"] * len(specs), [blob] * len(specs), specs)
        assert ecs == [bb.ErrorCode.OK] * len(specs), ecs
        assert np.array_equal(raw, want), np.nonzero(raw != want)[0][:8]
        assert _counter(cl, "device_get_strided_scatter_total") == len(specs)
        assert _counter(cl, "device_get_host_staged_total") >= 2  # the unaligned ones
        # dst width == dst pitch is the strided get
        dense, base = _buffer(10 * 4096)
        assert cl.batch_get_device_strided_scatter(["s"], [dense.ctypes.data + base], [64], [4096], [8192], [10], [4096], [4096], 0) == [bb.ErrorCode.OK]
        x, _ = model_pairs(64, 4096, 8192, 10, 4096, 4096, 0)
        assert np.array_equal(dense[base:base + 10 * 4096], blob[x])


def test_client_refusals_fail_alone(bb):
    with LocalCluster(cluster_id="slicerr", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        size = 100000
        blob = np.frombuffer(os.urandom(size), dtype=np.uint8).copy()
        assert cl.batch_put_device(["e"], [blob.ctypes.data], [size], _cfg(bb, 1, 2), 0) == [bb.ErrorCode.OK]
        E = bb.ErrorCode
        raw, base = _buffer(1 << 20)
        p = raw.ctypes.data + base
        cases = [((0, 100, 100, 1, 0, 16), E.INVALID_ARGUMENT),         # a zero destination width
                 ((0, 100, 100, 1, 64, 32), E.INVALID_ARGUMENT),        # destination rows wider than their pitch
                 ((0, 100, 50, 3, 64, 128), E.INVALID_ARGUMENT),        # window rows wider than their pitch
                 ((size - 10, 20, 20, 1, 64, 128), E.VALUE_OUT_OF_RANGE),
                 ((0, 2**40, 2**40, 2**30, 64, 128), E.VALUE_OUT_OF_RANGE),
                 ((0, 0, 0, 1, 0, 0), E.OK),                            # nothing to read
                 ((16, 64, 128, 4, 32, 48), E.OK)]
        keys = ["e"] * len(cases) + ["missing"]
        specs = [s for s, _ in cases] + [(0, 16, 16, 1, 16, 32)]
        ecs = cl.batch_get_device_strided_scatter(keys, [p] * len(keys), *[[s[k] for s in specs] for k in range(6)], 0)
        assert ecs == [e for _, e in cases] + [E.OBJECT_NOT_FOUND], ecs
        x, d = model_pairs(16, 64, 128, 4, 32, 48, 0)
        assert np.array_equal(raw[base + d], blob[x])
        want = np.full_like(raw, GUARD)
        want[base + d] = blob[x]
        assert np.array_equal(raw, want)
        # arity
        assert cl.batch_get_device_strided_scatter(["e"], [p], [0], [1], [1], [1], [], [], 0) == [E.INVALID_PARAMETERS]


def test_a_corrupt_copy_fails_over(bb):
    with LocalCluster(cluster_id="slicefo", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        size = 300000
        blob = np.frombuffer(os.urandom(size), dtype=np.uint8).copy()
        assert cl.batch_put_device(["f"], [blob.ctypes.data], [size], _cfg(bb, 2, 1), 0) == [bb.ErrorCode.OK]
        pools = {pl.id: pl for pl in cl.keystone().get_memory_pools()}
        for cp in cl.get_workers("f"):  # corrupt the first copy, in a gap of the window
            sh = cp.shards[0]
            w = [w for w in c.workers if w.backend(sh.pool_id) is not None][0]
            off = sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr + 5000
            b = w.backend(sh.pool_id)
            b.write(off, bytes([b.read(off, 1)[0] ^ 0xFF]))
            break
        spec = (64, 1024, 4096, 50, 512, 1024, 0)
        ecs, raw, want = _slice_gets(bb, cl, ["f"], [blob], [spec])
        assert ecs == [bb.ErrorCode.OK]
        assert np.array_equal(raw, want)
        assert _counter(cl, "replica_failover_total") + _counter(cl, "checksum_mismatch_total") >= 1


def test_client_fp8_slice_gets(bb):
    with LocalCluster(cluster_id="slicefp8", n_workers=2, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        rng = np.random.default_rng(0)
        n = 64 * 1024
        for wide, dt, es in ((bb.MxWide.BF16, np.uint16, 2), (bb.MxWide.F32, np.float32, 4)):
            if dt is np.uint16:
                src = (rng.standard_normal(n).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
            else:
                src = rng.standard_normal(n).astype(np.float32)
            key = f"p{es}"
            cfg = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_CPU])
            assert cl.batch_put_device_fp8([key], [src.ctypes.data], [n], cfg, 0, wide=wide) == [bb.ErrorCode.OK]
            whole = np.zeros(n, dtype=dt)
            assert cl.batch_get_device_fp8([key], [whole.ctypes.data], [n], 0, wide=wide) == [bb.ErrorCode.OK]
            # (offset, width, pitch, rows, dst width, dst pitch) in elements; 16-byte congruent destinations
            g = 16 // es
            specs = [(8 * g, 256, 1024, 40, 256, 256 + 4 * g), (0, 5000, 5000, 1, 1000, 1000 + g), (g, 64, 128, 100, 32, 32 + 2 * g)]
            for off, w, p, r, dw, dp in specs:
                out = np.full(es * (r * w // dw * dp + 2 * dp + 64), 0x5A, dtype=np.uint8).view(dt)
                base = (-out.ctypes.data % 16) // es
                ecs = cl.batch_get_device_fp8_strided_scatter([key], [out.ctypes.data + es * base], [n], [off], [w], [p], [r], [dw], [dp],
                                                              0, wide=wide)
                assert ecs == [bb.ErrorCode.OK], (es, off, ecs)
                x, d = model_pairs(off, w, p, r, dw, dp, 0)
                want = np.full_like(out, np.full(1, 0x5A5A5A5A, dtype=np.uint32).view(np.uint8)[:es].view(dt)[0])
                want[base + d] = whole[x]
                assert np.array_equal(out.view(np.uint8), want.view(np.uint8)), (es, off)
            # a window that holds the whole object (one range, and rows that touch) into rows, in one call with a
            # partial window: the whole object lands in the rows and the partial item is not disturbed
            calls = [(0, n, n, 1, 1024, 1024 + g), (0, 512, 512, n // 512, 4096, 4096 + 2 * g), (8 * g, 256, 1024, 40, 256, 256 + 4 * g)]
            outs, bases = [], []
            for off, w, p, r, dw, dp in calls:
                outs.append(np.full(es * (r * w // dw * dp + 2 * dp + 64), 0x5A, dtype=np.uint8).view(dt))
                bases.append((-outs[-1].ctypes.data % 16) // es)
            ecs = cl.batch_get_device_fp8_strided_scatter([key] * len(calls), [o.ctypes.data + es * b for o, b in zip(outs, bases)],
                                                          [n] * len(calls), *[[c[j] for c in calls] for j in range(6)], 0, wide=wide)
            assert ecs == [bb.ErrorCode.OK] * len(calls), (es, ecs)
            for out, base, (off, w, p, r, dw, dp) in zip(outs, bases, calls):
                x, d = model_pairs(off, w, p, r, dw, dp, 0)
                want = np.full_like(out, np.full(1, 0x5A5A5A5A, dtype=np.uint32).view(np.uint8)[:es].view(dt)[0])
                want[base + d] = whole[x]
                assert np.array_equal(out.view(np.uint8), want.view(np.uint8)), (es, off, w)
            # misaligned: no host-staged path for packed gets
            out = np.zeros(4096, dtype=dt)
            base = (-out.ctypes.data % 16) // es
            ecs = cl.batch_get_device_fp8_strided_scatter([key], [out.ctypes.data + es * (base + 1)], [n], [0], [64], [128], [4], [64],
                                                          [64 + g], 0, wide=wide)
            assert ecs == [bb.ErrorCode.NOT_IMPLEMENTED]
            assert not out.any()


def test_tensor_store_checks_come_before_any_transfer(bb):
    torch = pytest.importorskip("torch")
    from blackbird_b200.ops.tensor_store import TensorStore

    with LocalCluster(cluster_id="slicets", n_workers=1, pool_bytes=16 * MiB) as c:
        cl = make_client(bb, c)
        ts = TensorStore(cl)
        meta = b'{"dtype": "float32", "shape": [8, 16], "packed": null, "numel": 128}'
        assert cl.batch_put(["t#meta"], [meta], _cfg(bb, 1, 1, "CRC32C")) == [bb.ErrorCode.OK]
        out = torch.zeros(8, 4)
        with pytest.raises(KeyError):
            ts.get_slice_into("missing", out, 1, 0, 4)
        with pytest.raises(IndexError):
            ts.get_slice_into("t", out, 2, 0, 4)
        with pytest.raises(IndexError):
            ts.get_slice_into("t", out, 1, 3, 20)
        with pytest.raises(TypeError):
            ts.get_slice_into("t", out.double(), 1, 0, 4)
        with pytest.raises(ValueError):
            ts.get_slice_into("t", torch.zeros(8, 5), 1, 0, 4)
        with pytest.raises(ValueError):  # a CPU tensor
            ts.get_slice_into("t", out, -1, 0, 4)
        with pytest.raises(ValueError):
            ts.get_rows_into("t", torch.zeros(3, 16), 0, 4)
        with pytest.raises(ValueError):
            ts.batch_get_slices_into(["t"], [out, out], [1], [0], [4])
        assert not out.any()
