"""Packed puts of sliced bf16 tensors on the GPU: the gathering load of the fused pack kernel (bb_xfer_fp8 with XFER_GATHER)
through XferEngine.run_fp8, the client's batch_put_device_fp8_strided on a GpuRankCluster, and TensorStore.put(...,
pack_fp8=True) of slices.  A gathered item reads its elements from rows of a strided bf16 source (SourceRows,
common/store_window.h); the bf16 tile in shared memory is the tile of the compacted rows, so every check compares the
stored packed bytes with mxfp8_pack_ref of the numpy compaction, the guard bytes around every destination, and the digest,
which must equal bbh64 of the packed bytes and that of an unpatterned put of the compacted rows."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

T = 16384  # elements per payload tile (32 KiB of bf16)
MiB = 1 << 20
GUARD = 0xA5
GRIDS = [1, 7, "sms", "2sms"]


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need CUDA (marked gpu)")


@pytest.fixture(scope="module")
def _engine():
    from blackbird_b200 import _bb

    return _bb.XferEngine(0, 4096, 2)


@pytest.fixture
def eng(_engine):
    yield _engine
    _engine.set_max_ctas(0)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _grid(g):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return {"sms": sms, "2sms": 2 * sms}.get(g, g)


def source_index(n, pitch, width, phase):
    """Source element (from the pattern's row 0) of each object element: the rule of SourceRows."""
    y = np.arange(n, dtype=np.int64) + phase
    return y // width * pitch + y % width


class Puts:
    """Pack items gathered from one random bf16 source (the gaps hold random values too) or read contiguously, each into
    1-3 packed destinations, every destination a region of one guard-filled byte buffer.  An item is (n_elems, pattern
    (pitch, width, phase) in elements or None, ndst); each gathered source starts where 2 * (start + phase) is 16-byte
    aligned."""

    def __init__(self, bb, specs, seed=11):
        self.bb, self.specs = bb, specs
        rng = np.random.default_rng(seed)
        starts, idx, o = [], [], 64
        for n, pat, _ in specs:
            ix = source_index(n, *pat) if pat else np.arange(n, dtype=np.int64)
            o = (o + 7) // 8 * 8 + ((8 - pat[2] % 8) % 8 if pat else 0)
            starts.append(o)
            idx.append(ix)
            o += int(ix.max()) + 1 + 64
        host = ((rng.standard_normal(o + 64) * 3).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
        host[:4096] = 0  # all-zero blocks (scale 0) in the first objects
        self.src = torch.from_numpy(host.view(np.int16).copy()).cuda()
        self.dense = [host[s + ix] for s, ix in zip(starts, idx)]
        self.packed = [np.frombuffer(bb.mxfp8_pack_ref(d), dtype=np.uint8) for d in self.dense]
        self.digests = [bb.bbh64(p) for p in self.packed]
        self.regions, o = [], 64
        for (n, _, ndst), p in zip(specs, self.packed):
            rs = []
            for _ in range(ndst):
                rs.append(o)
                o = (o + p.size + 64 + 15) // 16 * 16
            self.regions.append(rs)
        self.dst = torch.full((o + 64,), GUARD, dtype=torch.uint8, device="cuda")
        self.items = []
        for (n, pat, _), s, rs in zip(specs, starts, self.regions):
            it = (self.src.data_ptr() + 2 * s, [self.dst.data_ptr() + r for r in rs], n)
            self.items.append(it + (None, None, pat) if pat else it)

    def check(self, what):
        torch.cuda.synchronize()
        want = np.full(self.dst.numel(), GUARD, dtype=np.uint8)
        for p, rs in zip(self.packed, self.regions):
            for r in rs:
                want[r:r + p.size] = p
        got = self.dst.cpu().numpy()
        if not np.array_equal(got, want):
            pytest.fail(f"{what}: bytes differ at {np.nonzero(got != want)[0][:8].tolist()}")


def patterns():
    """(n_elems, (pitch, width, phase), ndst): widths of 8 (2048 rows per tile), 40, 128 (a KV head), 1000, one tile and
    more than a tile; pitches below, at and above a tile; heads and tails (2 * phase no multiple of 16); objects of one
    tile, of one partial tile only and with a partial last tile."""
    return [(T, (64, 8, 0), 1), (4 * T + 96, (16, 8, 3), 2), (3 * T + 64, (48, 40, 5), 3), (8 * T, (1024, 128, 0), 1),
            (2 * T + 32, (1008, 1000, 999), 2), (3 * T, (T + 8, T, 0), 1), (5 * T + 32, (2 * T + 64, T + 40, 7), 3),
            (4 * T, (T, T - 64, 1), 1), (96, (40, 32, 0), 2), (T + 32, (136, 128, 127), 1)]


def test_gathered_packs_at_every_grid(bb, eng):
    """Every pattern with plain items mixed in, in batches of more than 8 items, at grids of 1, 7, the SM count and twice
    the SM count: the packed bytes in every replica equal the reference packing of the compaction, the guards are intact,
    and the digests equal bbh64 of the packed bytes and those of an unpatterned put of the compacted rows."""
    specs = patterns() + [(3 * T + 96, None, 2), (64, None, 1)]
    b = Puts(bb, specs)
    for g in GRIDS:
        eng.set_max_ctas(_grid(g))
        b.dst.fill_(GUARD)
        dg, st, _ = eng.run_fp8(b.items, False, _stream())
        assert st == [0] * len(specs) and dg == b.digests, g
        b.check(f"grid={g}")
    eng.set_max_ctas(0)
    dense = [torch.from_numpy(d.view(np.int16).copy()).cuda() for d in b.dense]
    outs = [torch.empty(p.size, dtype=torch.uint8, device="cuda") for p in b.packed]
    pdg, pst, _ = eng.run_fp8([(d.data_ptr(), o.data_ptr(), d.numel()) for d, o in zip(dense, outs)], False, _stream())
    assert pst == [0] * len(specs) and pdg == dg
    torch.cuda.synchronize()
    assert all(np.array_equal(o.cpu().numpy(), p) for o, p in zip(outs, b.packed))


def test_inline_sized_batches_mix_gathered_and_plain(bb, eng):
    """Batches of a few items, one of them a partial tile only, at every grid."""
    specs = [(4 * T, (2048, 512, 0), 3), (T + 32, None, 1), (32, (16, 8, 4), 1), (2 * T, (T + 16, 24, 23), 2)]
    for g in GRIDS:
        eng.set_max_ctas(_grid(g))
        b = Puts(bb, specs, seed=3)
        dg, st, _ = eng.run_fp8(b.items, False, _stream())
        assert st == [0] * len(specs) and dg == b.digests, g
        b.check(f"small grid={g}")


def test_rejected_gathers(bb, eng):
    src = torch.zeros(8 * T, dtype=torch.int16, device="cuda")
    slab = torch.full((4 * T,), GUARD, dtype=torch.uint8, device="cuda")
    s, d = src.data_ptr(), slab.data_ptr()
    n = 2 * T
    bad = [(([(s, d, n, None, None, (100, 0, 0))], False), "INVALID_ARGUMENT"),             # width 0
           (([(s, d, n, None, None, (100, 101, 0))], False), "INVALID_ARGUMENT"),           # width > pitch
           (([(s, d, n, None, None, (100, 48, 48))], False), "INVALID_ARGUMENT"),           # phase >= width
           (([(s, d, n, None, None, (2**62, 8, 0))], False), "INVALID_ARGUMENT"),           # pitch overflows its bytes
           (([(s, d, n, None, None, (64, 8, 0))], True), "INVALID_ARGUMENT"),               # a pattern on an unpack
           (([(s, d, n, None, None, (64, 8, 3))], False), "INVALID_ADDRESS"),               # src + 2 * phase 6 bytes off
           (([(s + 2, d, n, None, None, (64, 8, 0))], False), "INVALID_ADDRESS"),           # src 2 bytes off
           (([(s, d, n, None, None, (44, 40, 0))], False), "INVALID_ADDRESS"),              # gap of 4 elements
           (([(s, d + 8, n, None, None, (48, 40, 0))], False), "INVALID_ADDRESS")]          # packed object misaligned
    for (items, unpack), err in bad:
        with pytest.raises(RuntimeError, match=err):
            eng.run_fp8(items, unpack, _stream())
    torch.cuda.synchronize()
    assert bool((slab == GUARD).all())
    # an object inside one row may leave any gap: only src + 2 * phase has to be aligned
    src[:200] = torch.arange(200, dtype=torch.int16, device="cuda") * 37
    dg, st, _ = eng.run_fp8([(s - 8, d, 32, None, None, (100, 64, 4))], False, _stream())
    torch.cuda.synchronize()
    packed = np.frombuffer(bb.mxfp8_pack_ref(src[:32].cpu().numpy().view(np.uint16)), dtype=np.uint8)
    assert st == [0] and dg == [bb.bbh64(packed)]
    assert np.array_equal(slab[:packed.size].cpu().numpy(), packed) and bool((slab[packed.size:] == GUARD).all())


# ---------------------------------------------------------------------------------------------------- client


def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


def _cfg(bb, replicas=1):
    return bb.WorkerConfig(replication_factor=replicas, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_GPU])


def _flip(cl, sh, pos):
    be = cl.worker.backend(sh.pool_id)
    be.write(sh.offset + pos, bytes([be.read(sh.offset + pos, 1)[0] ^ 0xFF]))


def _sums(cl, key):
    return [[sh.checksum for sh in cp.shards] for cp in cl.client.get_workers(key)]


def _rows(t, off, width, pitch, rows):
    return t[off:off + (rows - 1) * pitch + width].unfold(0, width, pitch).reshape(-1) if rows > 1 else t[off:off + width]


def _ref(bb, dense):
    """The bf16 (int16) result of a fused get of dense packed: the reference unpack of its reference packing."""
    x = dense.cpu().numpy().view(np.uint16)
    return torch.from_numpy(np.frombuffer(bb.mxfp8_unpack_ref(bb.mxfp8_pack_ref(x), x.size), dtype=np.int16).copy()).cuda()


def test_client_fp8_strided_puts_read_back_through_every_fp8_get(bb):
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=128 << 20, cluster_id="t-fp8sput")
    try:
        g = torch.Generator(device="cuda").manual_seed(5)
        src = torch.randn(4 * MiB, device="cuda", generator=g).to(torch.bfloat16).view(torch.int16)
        before = src.clone()
        E = bb.ErrorCode
        # (source element offset, width, pitch, rows) in elements
        items = [(0, 128, 1024, 512), (8, 8, 64, 4096), (16, 1000, 1008, 64), (24, T + 40, T + 48, 4), (0, 96, 96, 100),
                 (40, 3008, 1, 1)]
        keys = [f"p{j}" for j in range(len(items))]
        n0, b0 = _counter(cl.client, "device_put_fp8_strided_total"), _counter(cl.client, "device_put_fp8_strided_bytes_total")
        l0 = cl.fabric.launches
        ecs = cl.client.batch_put_device_fp8_strided(keys, [src.data_ptr() + 2 * o for o, *_ in items], [i[1] for i in items],
                                                     [i[2] for i in items], [i[3] for i in items], _cfg(bb), _stream())
        assert ecs == [E.OK] * len(items), ecs
        assert cl.fabric.launches == l0 + 2  # the fused kernel and the scales batch
        assert _counter(cl.client, "device_put_fp8_strided_total") == n0 + len(items)
        assert _counter(cl.client, "device_put_fp8_strided_bytes_total") == b0 + sum(2 * w * r for _, w, _, r in items)
        for k, (o, w, p, r) in zip(keys, items):
            dense = _rows(src, o, w, p, r).contiguous()
            n, ref = dense.numel(), _ref(bb, dense)
            assert cl.client.batch_put_device_fp8([k + "/c"], [dense.data_ptr()], [n], _cfg(bb), _stream()) == [E.OK]
            assert _sums(cl, k) == _sums(cl, k + "/c"), k
            whole = torch.empty(n, dtype=torch.int16, device="cuda")
            part = torch.empty(n // 2 + 8, dtype=torch.int16, device="cuda")
            rows = torch.empty(n // 4 + 8, dtype=torch.int16, device="cuda")
            assert cl.client.batch_get_device_fp8([k], [whole.data_ptr()], [n], _stream()) == [E.OK]
            assert cl.client.batch_get_device_fp8_range([k], [part.data_ptr()], [n], [n // 4], [n // 2], _stream()) == [E.OK]
            assert cl.client.batch_get_device_fp8_strided([k], [rows.data_ptr()], [n], [0], [8], [32], [n // 32], _stream()) == [E.OK]
            torch.cuda.synchronize()
            assert torch.equal(whole, ref), k
            assert torch.equal(part[:n // 2], ref[n // 4:n // 4 + n // 2]), k
            assert torch.equal(rows[:n // 4], _rows(ref, 0, 8, 32, n // 32)), k
        assert torch.equal(src, before)
    finally:
        cl.stop()


def test_client_fp8_strided_put_two_copies_fail_over(bb):
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id="t-fp8sput-rep")
    try:
        g = torch.Generator(device="cuda").manual_seed(6)
        kv = torch.randn(256, 8, 128, device="cuda", generator=g).to(torch.bfloat16).view(torch.int16)
        view = kv[:, 2:4, :]
        n = view.numel()
        ecs = cl.client.batch_put_device_fp8_strided(["f"], [view.data_ptr()], [256], [1024], [256], _cfg(bb, 2), _stream())
        assert ecs == [bb.ErrorCode.OK]
        copies = cl.client.get_workers("f")
        assert len(copies) == 2 and all(len(c.shards) == 1 for c in copies)
        ref = _ref(bb, view.contiguous())
        fo = _counter(cl.client, "replica_failover_total")
        for sh in [c.shards[0] for c in copies]:  # one copy at a time is corrupt: exactly one of the two gets starts on it
            _flip(cl, sh, 300)
            out = torch.empty(n, dtype=torch.int16, device="cuda")
            assert cl.client.batch_get_device_fp8(["f"], [out.data_ptr()], [n], _stream()) == [bb.ErrorCode.OK]
            torch.cuda.synchronize()
            assert torch.equal(out, ref)
            _flip(cl, sh, 300)
        assert _counter(cl.client, "replica_failover_total") == fo + 1
    finally:
        cl.stop()


def test_client_fp8_strided_misaligned_item_fails_alone(bb):
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id="t-fp8sput-err")
    try:
        src = torch.randn(MiB, device="cuda").to(torch.bfloat16).view(torch.int16)
        E = bb.ErrorCode
        # (element offset, width, pitch, rows, expected)
        cases = [(0, 128, 1024, 64, E.OK), (1, 128, 1024, 64, E.NOT_IMPLEMENTED), (0, 40, 44, 32, E.NOT_IMPLEMENTED),
                 (0, 101, 100, 2, E.INVALID_ARGUMENT), (0, 8, 2**63, 3, E.VALUE_OUT_OF_RANGE), (8, 40, 48, 64, E.OK)]
        keys = [f"e{j}" for j in range(len(cases))]
        l0 = cl.fabric.launches
        ecs = cl.client.batch_put_device_fp8_strided(keys, [src.data_ptr() + 2 * c[0] for c in cases], [c[1] for c in cases],
                                                     [c[2] for c in cases], [c[3] for c in cases], _cfg(bb), _stream())
        assert ecs == [c[4] for c in cases], ecs
        assert cl.fabric.launches == l0 + 2
        for k, (o, w, p, r, e) in zip(keys, cases):
            assert cl.client.object_exists(k) == (e == E.OK), k
            if e == E.OK:
                dense = _rows(src, o, w, p, r)
                out = torch.empty(dense.numel(), dtype=torch.int16, device="cuda")
                assert cl.client.batch_get_device_fp8([k], [out.data_ptr()], [out.numel()], _stream()) == [E.OK]
                torch.cuda.synchronize()
                assert torch.equal(out, _ref(bb, dense)), k
    finally:
        cl.stop()


# ---------------------------------------------------------------------------------------------------- TensorStore


def test_tensor_store_packs_slices_in_place(bb):
    """put(view, pack_fp8=True) of KV heads, weight columns and t[::2] stores what put(view.contiguous(), pack_fp8=True)
    stores (the same get result, bit for bit, and the same recorded digest), through the gathered put and without
    allocating a contiguous temporary."""
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id="t-fp8sput-store")
    try:
        store = TensorStore(cl.client)
        g = torch.Generator(device="cuda").manual_seed(9)
        kv = torch.randn(2048, 8, 128, device="cuda", generator=g).to(torch.bfloat16)
        w = torch.randn(1024, 2048, device="cuda", generator=g).to(torch.bfloat16)
        t = torch.randn(1024, 1024, device="cuda", generator=g).to(torch.bfloat16)
        views = {"kv/h0": kv[:, 0:1, :], "kv/h2-6": kv[:, 2:6, :], "w/cols": w[:, 256:768], "t/step": t[::2]}
        for k, v in views.items():
            assert store._gatherable(v) is not None, k
            n0 = _counter(cl.client, "device_put_fp8_strided_total")
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            store.put(k, v, pack_fp8=True)
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - base
            assert peak < v.numel() * v.element_size(), (k, peak)
            assert _counter(cl.client, "device_put_fp8_strided_total") == n0 + 1, k
            store.put(k + "/c", v.contiguous(), pack_fp8=True)
            assert _counter(cl.client, "device_put_fp8_strided_total") == n0 + 1, k
            assert _sums(cl, k) == _sums(cl, k + "/c"), k
            got, want = store.get(k), store.get(k + "/c")
            assert got.shape == v.shape and torch.equal(got.view(torch.int16), want.view(torch.int16)), k
        # a batch of a slice, a contiguous tensor and a slice with a 4-element row gap (copied first) is one call and one
        # launch: the last two go as one row each
        x = torch.randn(64, 260, device="cuda", generator=g).to(torch.bfloat16)
        batch = {"b/view": w[:64, 0:512], "b/whole": x[:, :256].contiguous(), "b/gap4": x[:, :256]}
        assert store._gatherable(batch["b/gap4"]) is None
        n0, l0 = _counter(cl.client, "device_put_fp8_strided_total"), cl.fabric.launches
        store.batch_put(list(batch), list(batch.values()), pack_fp8=True)
        assert _counter(cl.client, "device_put_fp8_strided_total") == n0 + 3
        assert cl.fabric.launches == l0 + 2  # the fused kernel and the scales batch
        for k, v in batch.items():
            store.put(k + "/c", v.contiguous(), pack_fp8=True)
            assert torch.equal(store.get(k).view(torch.int16), store.get(k + "/c").view(torch.int16)), k
            assert _sums(cl, k) == _sums(cl, k + "/c"), k
    finally:
        cl.stop()
