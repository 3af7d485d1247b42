"""Strided device puts on the GPU: the gathering load of bb_xfer (XFER_GATHER) through XferEngine, the client's
batch_put_device_strided on a GpuRankCluster, and TensorStore.put of sliced tensors, against numpy / torch compactions and
the CPU digest models.  A gathered descriptor reads its object's bytes from rows of a strided source; the tile in shared
memory is the tile of the dense object, so every check covers the stored bytes, the guard bytes around every
destination, and the digest, which must equal that of a plain put of the compacted bytes."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

T = 16384
MiB = 1 << 20
GUARD = 0xA5
ALGOS = ["NONE", "CRC32C", "BBH64", "XXH3"]
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


def _model(bb, algo):
    return {"NONE": lambda b: 0, "CRC32C": bb.crc32c, "BBH64": bb.bbh64, "XXH3": bb.xxh3t64}[algo]


def _random(bb, n, seed):
    t = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
    bb.random_fill(t.data_ptr(), t.numel(), seed, _stream())
    return t


def source_index(n, pitch, width, phase):
    """Source offset (from the pattern's row 0) of each object byte: the rule of SourceRows."""
    y = np.arange(n, dtype=np.int64) + phase
    return y // width * pitch + y % width


class Batch:
    """Items whose objects are gathered from one random source (the gaps between rows hold random bytes too) or read
    contiguously, into 1-3 destinations each, every destination a region of one guard-filled buffer.  An item is
    (nbytes, pattern (pitch, width, phase) or None, ndst); each gathered source starts where src + phase is 16-byte aligned
    unless `skew` moves it."""

    def __init__(self, bb, specs, algo, skew=0, seed=11):
        self.bb, self.specs = bb, specs
        self.idx, starts, o = [], [], 64
        for n, pat, _ in specs:
            ix = source_index(n, *pat) if pat else np.arange(n, dtype=np.int64)
            o = (o + 15) // 16 * 16 + ((16 - pat[2] % 16) % 16 + skew if pat else 0)
            starts.append(o)
            self.idx.append(ix)
            o += (int(ix.max()) + 1 if n else 0) + 64
        self.src = _random(bb, o + 64, seed)
        host = self.src.cpu().numpy()
        self.dense = [host[s + ix] for s, ix in zip(starts, self.idx)]
        self.regions, o = [], 64
        for n, _, ndst in specs:
            rs = []
            for _ in range(ndst):
                rs.append(o)
                o = (o + n + 64 + 15) // 16 * 16
            self.regions.append(rs)
        self.dst = torch.full((o + 64,), GUARD, dtype=torch.uint8, device="cuda")
        model = _model(bb, algo)
        self.digests = [model(d.tobytes()) for d in self.dense]
        self.items = []
        for (n, pat, _), s, rs in zip(specs, starts, self.regions):
            it = (self.src.data_ptr() + s, [self.dst.data_ptr() + r for r in rs], n, 0, 0)
            self.items.append(it + (0, None, pat) if pat else it)

    def check(self, what):
        torch.cuda.synchronize()
        want = np.full(self.dst.numel(), GUARD, dtype=np.uint8)
        for d, rs in zip(self.dense, self.regions):
            for r in rs:
                want[r:r + d.size] = d
        got = self.dst.cpu().numpy()
        if not np.array_equal(got, want):
            pytest.fail(f"{what}: bytes differ at {np.nonzero(got != want)[0][:8].tolist()}")


def patterns():
    """(nbytes, (pitch, width, phase), ndst): widths of 1 to 17 bytes, 4000, 16 KiB and above; pitches below, at and above
    16 KiB; heads and tails (phase not a multiple of 16); objects of 1 byte to several MiB."""
    return [(1, (17, 1, 0), 1), (7, (24, 8, 3), 2), (3000, (17, 1, 0), 3), (5000, (31, 15, 7), 1), (4096, (32, 16, 0), 2),
            (2 * T + 5, (33, 17, 16), 3), (3 * T + 1, (132, 100, 99), 1), (5 * T, (4016, 4000, 123), 2),
            (3 * T + 77, (T + 48, T, 5), 1), (2 * T, (2 * T + 19, T + 3, T), 3), (8 * T + 9, (40016, 40000, 0), 1),
            (4 * MiB, (128, 64, 0), 2), (6 * T + 11, (4096 + 16, 4096, 4000), 1)]


@pytest.mark.parametrize("algo", ALGOS)
def test_gathered_puts_at_every_grid(bb, eng, algo):
    """Every pattern in one device-table batch with plain items mixed in, at grids of 1, 7, the SM count and twice the SM
    count: the destinations equal the numpy compaction, the guards are intact, and the digests equal the CPU model of the
    compacted bytes and those of a plain put of them."""
    A = getattr(bb.ChecksumAlgo, algo)
    specs = patterns() + [(3 * T + 7, None, 2), (100, None, 1)]
    b = Batch(bb, specs, algo)
    for g in GRIDS:
        eng.set_max_ctas(_grid(g))
        b.dst.fill_(GUARD)
        dg, st, _ = eng.run(b.items, A, _stream())
        assert st == [0] * len(specs), (g, st)
        if algo != "NONE":
            assert dg == b.digests, g
        b.check(f"{algo} grid={g}")
    eng.set_max_ctas(0)
    # the same objects as plain puts of the compacted bytes: the same digests
    dense = [torch.from_numpy(d.copy()).cuda() if d.size else torch.empty(16, dtype=torch.uint8, device="cuda") for d in b.dense]
    outs = [torch.empty(max(d.numel(), 16), dtype=torch.uint8, device="cuda") for d in dense]
    plain = [(d.data_ptr(), o.data_ptr(), n) for d, o, (n, _, _) in zip(dense, outs, specs)]
    pdg, pst, _ = eng.run(plain, A, _stream())
    assert pst == [0] * len(specs) and (algo == "NONE" or pdg == dg)


@pytest.mark.parametrize("algo", ALGOS)
def test_inline_batches_mix_gathered_and_plain(bb, eng, algo):
    """Batches of <= 8 descriptors carry their source rows in the kernel parameters."""
    A = getattr(bb.ChecksumAlgo, algo)
    specs = [(3 * T + 7, (256, 128, 0), 1), (5000, None, 2), (2 * T + 1, (4113, 1, 0), 3), (100, (40, 24, 13), 1),
             (4 * T, (6000, 6000 - 16 * 7, 5), 2), (T, None, 1)]
    for g in GRIDS:
        eng.set_max_ctas(_grid(g))
        b = Batch(bb, specs, algo, seed=3)
        dg, st, _ = eng.run(b.items, A, _stream())
        assert st == [0] * len(specs)
        if algo != "NONE":
            assert dg == b.digests
        b.check(f"inline {algo} grid={g}")


def test_small_gathered_items_take_the_fused_kernel(bb, eng):
    """Objects of 4 KiB and less, gathered, never take the warp-per-object kernel or the mailbox."""
    b = Batch(bb, [(4096, (64, 16, 0), 1), (100, (20, 4, 0), 1), (1, (17, 1, 0), 1)], "XXH3")
    sl, mb, la = eng.small_launches, eng.mailbox_requests, eng.launches
    dg, st, _ = eng.run(b.items, bb.ChecksumAlgo.XXH3, _stream())
    assert st == [0] * 3 and dg == b.digests
    assert eng.small_launches == sl and eng.mailbox_requests == mb and eng.launches == la + 1
    b.check("small")


def test_rejected_gathers(bb, eng):
    src = _random(bb, 4 * T, 1)
    dst = torch.full((2 * T,), GUARD, dtype=torch.uint8, device="cuda")
    s, d = src.data_ptr(), dst.data_ptr()
    A = bb.ChecksumAlgo.XXH3
    bad = [((s, d, 1000, 0, 0, 0, None, (100, 0, 0)), "INVALID_ARGUMENT"),                 # width 0
           ((s, d, 1000, 0, 0, 0, None, (100, 101, 0)), "INVALID_ARGUMENT"),               # width > pitch
           ((s, d, 1000, 0, 0, 0, None, (100, 50, 50)), "INVALID_ARGUMENT"),               # phase >= width
           ((s, d, 1000, 0, bb.XFER_GATHER), "INVALID_ARGUMENT"),                          # flag without a pattern
           ((s, d, 1000, 0, 0, 0, (0, 500), (96, 80, 0)), "INVALID_ARGUMENT"),             # with a window
           ((s, [], 1000, 0, bb.XFER_RAW_SUM, 0, None, (96, 80, 0)), "INVALID_ARGUMENT"),  # with RAW_SUM
           ((s, d, 1000, 0, 0, 0, None, (96, 80, 5)), "INVALID_ADDRESS"),                  # src + phase misaligned
           ((s + 8, d, 1000, 0, 0, 0, None, (96, 80, 0)), "INVALID_ADDRESS"),              # src misaligned
           ((s, d, 1000, 0, 0, 0, None, (100, 60, 0)), "INVALID_ADDRESS"),                 # gap of 40 bytes
           ((s, d + 8, 1000, 0, 0, 0, None, (96, 80, 0)), "INVALID_ADDRESS")]              # dst misaligned
    for it, err in bad:
        with pytest.raises(RuntimeError, match=err):
            eng.run([it], A, _stream())
    # a span inside one row may have any gap: only src + phase has to be aligned
    eng.run([(s - 4, d, 50, 0, 0, 0, None, (100, 60, 4))], A, _stream())
    torch.cuda.synchronize()
    assert torch.equal(dst[:50], src[:50]) and bool((dst[50:] == GUARD).all())


# ---------------------------------------------------------------------------------------------------- client


def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


def _cfg(bb, algo, replicas=1, tier="RAM_GPU"):
    return bb.WorkerConfig(replication_factor=replicas, max_workers_per_copy=1, ttl_ms=0, checksum=getattr(bb.ChecksumAlgo, algo),
                           preferred_classes=[getattr(bb.StorageClass, tier)])


def _rows(t, off, width, pitch, rows):
    return t[off:off + (rows - 1) * pitch + width].unfold(0, width, pitch).reshape(-1) if rows > 1 else t[off:off + width]


def _get(bb, cl, key, n):
    out = torch.full((n + 32,), GUARD, dtype=torch.uint8, device="cuda")
    ecs, sizes = cl.client.batch_get_device([key], [out.data_ptr()], [n], _stream())
    assert ecs == [bb.ErrorCode.OK] and sizes == [n], ecs
    torch.cuda.synchronize()
    assert bool((out[n:] == GUARD).all())
    return out[:n]


def _sums(cl, key):
    return [[sh.checksum for sh in cp.shards] for cp in cl.client.get_workers(key)]


@pytest.mark.parametrize("algo", ALGOS)
def test_client_strided_puts(bb, algo):
    """Objects in HBM, in a pinned DRAM pool, replicated, and striped over both (shard edges mid-row): one batch of strided
    puts is one launch; a get returns the compacted rows and every copy's checksums equal those of a contiguous put; a
    misaligned item is staged alone; the source is unchanged."""
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=128 << 20, cluster_id=f"t-sput-{algo}", dram_bytes=64 << 20, max_replicas=3)
    try:
        src = _random(bb, 8 * MiB, 41)
        before = src.clone()
        striped = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=2, ttl_ms=0, min_shard_size=4096,
                                  checksum=getattr(bb.ChecksumAlgo, algo), preferred_classes=[bb.StorageClass.RAM_GPU, bb.StorageClass.RAM_CPU])
        # (source offset, width, pitch, rows, config)
        items = [(0, 96, 128, 21845, striped),               # 2 MiB + change over two stripes, the edge mid-row
                 (16, 1, 17, 4000, _cfg(bb, algo)), (32, 4000, 4016, 300, _cfg(bb, algo, 2)),
                 (48, T, T + 48, 40, _cfg(bb, algo, 1, "RAM_CPU")), (0, 5000, 5000, 3, _cfg(bb, algo)),
                 (64, 3000, 9000, 1, _cfg(bb, algo))]
        keys = [f"s{j}" for j in range(len(items))]
        l0, st0 = cl.fabric.launches, _counter(cl.client, "device_put_host_staged_total")
        for k, (off, w, p, r, cfg) in zip(keys, items):  # one config per call: each call is one batch
            ecs = cl.client.batch_put_device_strided([k], [src.data_ptr() + off], [w], [p], [r], cfg, _stream())
            assert ecs == [bb.ErrorCode.OK], (k, ecs)
        assert _counter(cl.client, "device_put_host_staged_total") == st0
        assert cl.fabric.launches == l0 + len(items)
        assert [len(c.shards) for c in cl.client.get_workers("s0")] == [2]
        for k, (off, w, p, r, cfg) in zip(keys, items):
            dense = _rows(src, off, w, p, r).contiguous()
            assert torch.equal(_get(bb, cl, k, dense.numel()), dense), k
            ck = k + "/c"
            assert cl.client.batch_put_device([ck], [dense.data_ptr()], [dense.numel()], cfg, _stream()) == [bb.ErrorCode.OK]
            got, ref = _sums(cl, k), _sums(cl, ck)
            assert all(g == ref[0] for g in got) and len(got) == len(ref), (k, got, ref)
        # several objects in one call are one launch; a misaligned source and a 40-byte gap are staged alone
        pats = [(0, 100, 132, 500), (5, 100, 132, 500), (16, 24, 64, 700), (32, 48, 80, 900)]
        l0, st0 = cl.fabric.launches, _counter(cl.client, "device_put_host_staged_total")
        ks = [f"m{j}" for j in range(4)]
        ecs = cl.client.batch_put_device_strided(ks, [src.data_ptr() + p[0] for p in pats], [p[1] for p in pats], [p[2] for p in pats],
                                                 [p[3] for p in pats], _cfg(bb, algo), _stream())
        assert ecs == [bb.ErrorCode.OK] * 4
        assert cl.fabric.launches == l0 + 1 and _counter(cl.client, "device_put_host_staged_total") == st0 + 2
        for k, (off, w, p, r) in zip(ks, pats):
            dense = _rows(src, off, w, p, r)
            assert torch.equal(_get(bb, cl, k, dense.numel()), dense), k
        E = bb.ErrorCode
        ecs = cl.client.batch_put_device_strided(["e0", "e1", "e2"], [src.data_ptr()] * 3, [65, 8, 0], [64, 2**63, 64], [2, 3, 9],
                                                 _cfg(bb, algo), _stream())
        assert ecs == [E.INVALID_ARGUMENT, E.VALUE_OUT_OF_RANGE, E.OK], ecs
        torch.cuda.synchronize()
        assert torch.equal(src, before)
    finally:
        cl.stop()


# ---------------------------------------------------------------------------------------------------- TensorStore


def test_tensor_store_puts_slices_in_place(bb):
    """`put` of narrow views along every dim and of t[::2] is one gathered put (no contiguous copy) when the view is
    co-aligned, else a put of t.contiguous(); transposed views and pack_fp8 keep the copy.  Every stored tensor reads back
    through get, get_rows and get_slice as t.contiguous() would."""
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id="t-sput-store")
    try:
        store = TensorStore(cl.client)
        g = torch.Generator(device="cuda").manual_seed(9)
        views, fused = {}, 0
        for dt in (torch.bfloat16, torch.float32, torch.uint8):
            base = torch.randn(16, 12, 10, 64, device="cuda", generator=g).mul(40).to(dt)
            for d in range(base.dim()):
                n = base.shape[d]
                for a, b in ((0, n // 2), (n // 4, n), (1, n - 1)):
                    views[f"{dt}/{d}/{a}"] = base.narrow(d, a, b - a)
            views[f"{dt}/step"] = base[::2]
            views[f"{dt}/T"] = base[0, 0].t()  # transposed: copied
        for t in views.values():
            fused += int(store._gatherable(t) is not None)
        snapshot = {k: v.clone() for k, v in views.items()}
        n0 = _counter(cl.client, "device_put_strided_total")
        store.batch_put(list(views), list(views.values()))
        assert _counter(cl.client, "device_put_strided_total") - n0 == len(views)  # one call for the whole batch
        assert fused >= 12, fused
        for k, v in views.items():
            want = v.contiguous()
            assert torch.equal(v, snapshot[k])
            got = store.get(k)
            assert got.dtype == want.dtype and got.shape == want.shape and torch.equal(got, want), k
            n = want.shape[0]
            assert torch.equal(store.get_rows(k, n // 3, n), want[n // 3:]), k
            d = want.dim() - 1
            assert torch.equal(store.get_slice(k, d, 1, want.shape[d]), want.narrow(d, 1, want.shape[d] - 1).contiguous()), k
        # one view put alone, and a single tensor that is contiguous: the plain put
        x = torch.randn(64, 256, device="cuda", generator=g).to(torch.bfloat16)
        n0 = _counter(cl.client, "device_put_strided_total")
        store.put("cols", x[:, 64:192])
        store.put("whole", x)
        assert _counter(cl.client, "device_put_strided_total") == n0 + 1
        assert torch.equal(store.get("cols"), x[:, 64:192].contiguous()) and torch.equal(store.get("whole"), x)
        # MXFP8 packing takes the copy
        store.put("packed", x[:, 64:192], pack_fp8=True)
        assert _counter(cl.client, "device_put_strided_total") == n0 + 1
        ref = x[:, 64:192].contiguous()
        store.put("packed_ref", ref, pack_fp8=True)
        assert torch.equal(store.get("packed").view(torch.int16), store.get("packed_ref").view(torch.int16))
    finally:
        cl.stop()
