"""Byte-range device gets on the GPU: the store window of bb_xfer (XFER_WINDOW) through XferEngine, the client's
batch_get_device_range on a GpuRankCluster, and TensorStore.get_rows, against numpy / torch slices and the CPU digest
models.  A windowed descriptor reads and hashes its whole object and stores only the window, so every check covers the
stored bytes, the guard bytes around every window, the digest and the verify status."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

T = 16384
MiB = 1 << 20
GUARD = 0xA5
ALGOS = ["NONE", "CRC32C", "BBH64", "XXH3"]
GRIDS = [1, 7, "sms", "2sms"]
SIZES = [1, 15, 16, 4096, 4097, T, T + 1, 3 * T + 7, 64 * MiB + 5]


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
    _engine.set_tile_trace(False)


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


def windows(n):
    """Windows of an n-byte object: empty, whole, inside one tile, across a tile edge, lo / hi on a tile edge and one byte
    either side of it, inside the last partial tile, and lo % 16 in {0, 1, 8, 15}."""
    last = (n - 1) // T * T
    cand = [(0, 0), (n // 2, n // 2), (n, n), (0, n), (min(5, n), min(n, 100)), (T - 7, T + 9),
            (T - 1, n), (T, n), (T + 1, n), (0, T - 1), (0, T), (0, T + 1), (2 * T - 1, 2 * T + 1),
            (last + 1, n - 1), (last, n), (16, n), (1, n), (8, n - 3), (15, n - 1), (17, 17 + 4096), (n - 1, n)]
    out = []
    for w in cand:
        if 0 <= w[0] <= w[1] <= n and w not in out:
            out.append(w)
    return out


class Batch:
    """Items reading objects of `src` (object i at src_offs[i], n[i] bytes) into one guard-filled destination buffer: item
    k stores window w[k] (or, for None, the whole object) at its own region, congruent to lo mod 16, with guard bytes
    around it."""

    def __init__(self, bb, src, src_offs, sizes, wins, algo, verify=True, expect=None):
        self.bb, self.src, self.src_offs, self.sizes, self.wins = bb, src, src_offs, sizes, wins
        self.regions, o = [], 64
        for n, w in zip(sizes, wins):
            lo, hi = w if w is not None else (0, n)
            o = (o + 15) // 16 * 16 + lo % 16
            self.regions.append(o)
            o += hi - lo + 64
        self.dst = torch.full((o + 64,), GUARD, dtype=torch.uint8, device="cuda")
        model = _model(bb, algo)
        host = src.cpu().numpy()
        self.digests = [model(host[so:so + n]) for so, n in zip(src_offs, sizes)] if expect is None else expect
        self.items = []
        for so, n, w, r, d in zip(src_offs, sizes, wins, self.regions, self.digests):
            flags = bb.XFER_VERIFY if (verify and algo != "NONE") else 0
            lo = w[0] if w is not None else 0
            it = (src.data_ptr() + so, self.dst.data_ptr() + r - lo, n, d, flags)
            self.items.append(it if w is None else it + (0, w))

    def want(self):
        want = torch.full_like(self.dst, GUARD)
        for so, n, w, r in zip(self.src_offs, self.sizes, self.wins, self.regions):
            lo, hi = w if w is not None else (0, n)
            want[r:r + hi - lo] = self.src[so + lo:so + hi]
        return want

    def check(self, what):
        torch.cuda.synchronize()
        want = self.want()
        if not torch.equal(self.dst, want):
            bad = (self.dst != want).nonzero().flatten()[:8].tolist()
            pytest.fail(f"{what}: bytes differ at {bad}; regions {self.regions[:8]}")


@pytest.mark.parametrize("algo", ALGOS)
def test_windows_at_every_object_size_and_grid(bb, eng, algo):
    """Every window shape of every object size, one batch per size (a device-table batch: more than 8 items, whole
    objects mixed in), at grids of 1, 7, the SM count and twice the SM count, so that windows straddle CTA runs."""
    A = getattr(bb.ChecksumAlgo, algo)
    for n in SIZES:
        src = _random(bb, n, n)
        ws = windows(n)
        ws = ws[:3] + [None] + ws[3:] + [None]
        ws += [None] * (9 - len(ws))
        b = Batch(bb, src, [0] * len(ws), [n] * len(ws), ws, algo)
        assert len(ws) > 8
        for g in GRIDS if n < 64 * MiB else [1, "sms"]:
            eng.set_max_ctas(_grid(g))
            b.dst.fill_(GUARD)
            dg, st, _ = eng.run(b.items, A, _stream())
            assert st == [0] * len(ws), (n, g, st)
            if algo != "NONE":
                assert dg == b.digests, (n, g)
            b.check(f"{algo} n={n} grid={g}")


@pytest.mark.parametrize("algo", ALGOS)
def test_inline_batches_mix_windows_and_whole_objects(bb, eng, algo):
    """Batches of <= 8 descriptors travel in the kernel parameters: windowed and whole items side by side, with the same
    digest and status as a plain verified get of the same objects."""
    A = getattr(bb.ChecksumAlgo, algo)
    sizes = [3 * T + 7, 5000, T + 1, 100, 2 * T]
    offs = [0, 65536, 131072, 196608, 262144]
    src = _random(bb, 300000, 7)
    wins = [(T - 1, 2 * T + 3), None, (1, T), None, (8, 8)]
    b = Batch(bb, src, offs, sizes, wins, algo)
    dg, st, _ = eng.run(b.items, A, _stream())
    b.check("inline")
    plain = Batch(bb, src, offs, sizes, [None] * 5, algo)
    pdg, pst, _ = eng.run(plain.items, A, _stream())
    assert st == pst == [0] * 5 and dg == pdg


@pytest.mark.parametrize("algo", ["CRC32C", "BBH64", "XXH3", "NONE"])
def test_a_flipped_byte_outside_the_window_fails_verification(bb, eng, algo):
    A = getattr(bb.ChecksumAlgo, algo)
    n = 3 * T + 7
    src = _random(bb, n, 3)
    good = _model(bb, algo)(src.cpu().numpy())
    src[100] ^= 0xFF  # outside every window below
    for w in [(20000, 30000), (T, 2 * T), (n - 1, n), (5000, 5000)]:
        b = Batch(bb, src, [0], [n], [w], algo, expect=[good])
        _, st, _ = eng.run(b.items, A, _stream())
        assert st == [0 if algo == "NONE" else 1], (w, st)
        b.check("the window is stored even when the object fails verification")


def test_none_reads_only_the_trimmed_span(bb, eng):
    """Without a checksum the engine trims a windowed descriptor to [lo & ~15, hi): the tile trace holds 4 entries per
    tile of the trimmed descriptors, and empty windows read nothing."""
    n = 10 * T + 5
    src = _random(bb, n, 9)
    wins = [(5 * T + 3, 5 * T + 40), (T - 1, 3 * T + 1), (0, n), (7, 7), (9 * T + 17, n)]
    b = Batch(bb, src, [0] * len(wins), [n] * len(wins), wins, "NONE")
    eng.set_tile_trace(True)
    _, st, _ = eng.run(b.items, bb.ChecksumAlgo.NONE, _stream())
    tiles = sum(-(-(hi - (lo & ~15)) // T) for lo, hi in wins if hi > lo)
    assert st == [0] * len(wins) and len(eng.tile_trace()) == 4 * tiles
    b.check("trimmed")
    # XXH3 reads every tile of every non-empty object
    b = Batch(bb, src, [0] * len(wins), [n] * len(wins), wins, "XXH3")
    eng.run(b.items, bb.ChecksumAlgo.XXH3, _stream())
    assert len(eng.tile_trace()) == 4 * len(wins) * (-(-n // T))
    b.check("verified")


def test_windowed_small_items_take_the_fused_kernel(bb, eng):
    src = _random(bb, 8 * 4096, 5)
    for algo in ("CRC32C", "XXH3", "NONE"):
        A = getattr(bb.ChecksumAlgo, algo)
        b = Batch(bb, src, [4096 * i for i in range(3)], [4096, 100, 4000], [(1, 4095), (0, 50), None], algo)
        sl, mb, la = eng.small_launches, eng.mailbox_requests, eng.launches
        _, st, _ = eng.run(b.items, A, _stream())
        assert st == [0] * 3 and eng.small_launches == sl and eng.mailbox_requests == mb and eng.launches == la + 1
        b.check(algo)


def test_rejected_windows(bb, eng):
    src = _random(bb, 2 * T, 1)
    dst = torch.full((2 * T,), GUARD, dtype=torch.uint8, device="cuda")
    s, d = src.data_ptr(), dst.data_ptr()
    A = bb.ChecksumAlgo.XXH3
    bad = [((s, d, 1000, 0, 0, 0, (10, 5)), "INVALID_ARGUMENT"),                       # lo > hi
           ((s, d, 1000, 0, 0, 0, (0, 1001)), "INVALID_ARGUMENT"),                     # past the object
           ((s, [d, d + 4096], 1000, 0, 0, 0, (0, 10)), "INVALID_ARGUMENT"),           # two destinations
           ((s, d, 1024, 0, bb.XFER_MULTIMEM, 0, (0, 10)), "INVALID_ARGUMENT"),        # multicast
           ((s, [], 1000, 0, bb.XFER_RAW_SUM, 0, (0, 10)), "INVALID_ARGUMENT"),        # hash-only slice
           ((s, d + 8, 1000, 0, 0, 0, (8, 100)), "INVALID_ADDRESS")]                   # dst[0] not 16-byte aligned
    for it, err in bad:
        with pytest.raises(RuntimeError, match=err):
            eng.run([it], A, _stream())
    torch.cuda.synchronize()
    assert bool((dst == GUARD).all())


def test_window_past_4_gib(bb, eng):
    """One engine item of 2^32 + 16385 bytes whose window lies past 2^32: 64-bit window bounds and store offsets."""
    big = (1 << 32) + 16385
    src = _random(bb, big, 61)
    try:
        host = src.cpu().numpy()
        want = bb.xxh3t64(host)
        w = ((1 << 32) - 9, big - 3)
        b = Batch(bb, src, [0], [big], [w], "XXH3", expect=[want])
        dg, st, _ = eng.run(b.items, bb.ChecksumAlgo.XXH3, _stream())
        assert st == [0] and dg == [want]
        b.check("past 4 GiB")
    finally:
        del src
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------- client


def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


def _cfg(bb, algo, replicas=1, tier="RAM_GPU"):
    return bb.WorkerConfig(replication_factor=replicas, max_workers_per_copy=1, ttl_ms=0, checksum=getattr(bb.ChecksumAlgo, algo),
                           preferred_classes=[getattr(bb.StorageClass, tier)])


def _flip(bb, cl, sh, pos):
    be = cl.worker.backend(sh.pool_id)
    if sh.location["kind"] == "gpu":
        off = sh.offset
    else:
        pools = {p.id: p for p in cl.client.keystone().get_memory_pools()}
        off = sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr
    be.write(off + pos, bytes([be.read(off + pos, 1)[0] ^ 0xFF]))


def _range_get(cl, keys, ranges, skew=None):
    """Range gets into one guard-filled device buffer; returns (error codes, buffer, region offsets)."""
    regions, o = [], 256
    for i, (_, n) in enumerate(ranges):
        regions.append(o + (skew or {}).get(i, 0))
        o += (n + 255) // 256 * 256 + 256
    out = torch.full((o,), GUARD, dtype=torch.uint8, device="cuda")
    ecs = cl.client.batch_get_device_range(keys, [out.data_ptr() + r for r in regions], [a for a, _ in ranges], [n for _, n in ranges],
                                           _stream())
    return ecs, out, regions


def _check_ranges(out, regions, objs, ranges, ok):
    want = torch.full_like(out, GUARD)
    for r, obj, (a, n), good in zip(regions, objs, ranges, ok):
        if good:
            want[r:r + n] = obj[a:a + n]
    torch.cuda.synchronize()
    if not torch.equal(out, want):
        pytest.fail(f"range get wrote wrong bytes at {(out != want).nonzero().flatten()[:8].tolist()}")


@pytest.mark.parametrize("algo", ["XXH3", "CRC32C", "BBH64"])
def test_client_ranges_fail_over_from_a_copy_corrupt_outside_the_range(bb, algo):
    """Replication 1 to 3 on one slab (the client reads copy 0 first: every copy is local).  Copy 0 is corrupt outside the
    range: the range comes from a replica and the mismatch is counted; with one copy it fails."""
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=128 << 20, cluster_id=f"t-rng-rep-{algo}", max_replicas=3)
    try:
        n = 3 * T + 7
        src = _random(bb, n, 21)
        for rep in (1, 2, 3):
            key = f"r{rep}"
            assert cl.client.batch_put_device([key], [src.data_ptr()], [n], _cfg(bb, algo, rep), _stream()) == [bb.ErrorCode.OK]
            _flip(bb, cl, cl.client.get_workers(key)[0].shards[0], 5)
            r = (T + 16, T)  # 16-byte aligned offset: the fused path
            mm, l0 = _counter(cl.client, "checksum_mismatch_total"), cl.fabric.launches
            ecs, out, regions = _range_get(cl, [key], [r])
            ok = rep > 1
            assert ecs == [bb.ErrorCode.OK if ok else bb.ErrorCode.CHECKSUM_MISMATCH], (rep, ecs)
            assert _counter(cl.client, "checksum_mismatch_total") > mm
            if ok:
                _check_ranges(out, regions, [src], [r], [True])
                assert cl.fabric.launches == l0 + 2  # first read and one fail-over
    finally:
        cl.stop()


@pytest.mark.parametrize("algo", ALGOS)
def test_client_ranges_over_hbm_and_dram_in_one_launch(bb, algo):
    """Single-shard objects in this GPU's HBM slab and in a pinned DRAM pool: one batch of ranges (inside a tile, across
    tile edges, whole, empty) costs one launch; out-of-range and missing keys fail alone."""
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id=f"t-rng-tier-{algo}", dram_bytes=64 << 20)
    try:
        sizes = [5 * T + 11, 70001, 40001, 2 * MiB + 5]
        srcs = [_random(bb, n, 30 + i) for i, n in enumerate(sizes)]
        keys = []
        for i, (n, s) in enumerate(zip(sizes, srcs)):
            for tier in ("RAM_GPU", "RAM_CPU"):
                k = f"{tier}/{i}"
                assert cl.client.batch_put_device([k], [s.data_ptr()], [n], _cfg(bb, algo, 1, tier), _stream()) == [bb.ErrorCode.OK]
                keys.append((k, i))
        ks, objs, ranges = [], [], []
        for k, i in keys:
            n = sizes[i]
            for r in [(16, 100), (T - 16, 48), (0, n), (n - 32 - n % 16, 32 + n % 16), (32, 0)]:
                ks.append(k), objs.append(srcs[i]), ranges.append(r)
        l0, st0 = cl.fabric.launches, _counter(cl.client, "device_get_host_staged_total")
        ecs, out, regions = _range_get(cl, ks, ranges)
        assert ecs == [bb.ErrorCode.OK] * len(ks), ecs
        assert cl.fabric.launches == l0 + 1 and _counter(cl.client, "device_get_host_staged_total") == st0
        _check_ranges(out, regions, objs, ranges, [True] * len(ks))
        E = bb.ErrorCode
        ecs, out, regions = _range_get(cl, [keys[0][0], "missing", keys[1][0], keys[2][0]],
                                       [(0, sizes[0] + 1), (0, 16), (48, 64), (2**64 - 16, 32)])
        assert ecs == [E.VALUE_OUT_OF_RANGE, E.OBJECT_NOT_FOUND, E.OK, E.VALUE_OUT_OF_RANGE], ecs
        _check_ranges(out, regions, [srcs[0], None, srcs[0], None], [(0, 0), (0, 0), (48, 64), (0, 0)], [False, False, True, False])
    finally:
        cl.stop()


@pytest.mark.parametrize("algo", ["XXH3", "NONE"])
def test_client_stages_ranges_with_a_misaligned_virtual_base(bb, algo):
    """(ptr - offset) % 16 != 0 goes through the host (one staged object, counted); its neighbours still take one fused
    launch."""
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id=f"t-rng-al-{algo}")
    try:
        n = 200000
        src = _random(bb, n, 77)
        assert cl.client.batch_put_device(["a"], [src.data_ptr()], [n], _cfg(bb, algo), _stream()) == [bb.ErrorCode.OK]
        ranges = [(16, 5000), (7, 100), (20, 4000), (1, 33)]
        skew = {1: 7, 2: 7, 3: 1}  # (ptr - offset) % 16 = 0, 0, 3, 0
        l0, st0 = cl.fabric.launches, _counter(cl.client, "device_get_host_staged_total")
        ecs, out, regions = _range_get(cl, ["a"] * 4, ranges, skew)
        assert ecs == [bb.ErrorCode.OK] * 4
        assert cl.fabric.launches == l0 + 1 and _counter(cl.client, "device_get_host_staged_total") == st0 + 1
        _check_ranges(out, regions, [src] * 4, ranges, [True] * 4)
    finally:
        cl.stop()


# ---------------------------------------------------------------------------------------------------- TensorStore


def test_tensor_store_get_rows(bb):
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=128 << 20, cluster_id="t-rng-rows")
    try:
        store = TensorStore(cl.client)
        g = torch.Generator(device="cuda").manual_seed(5)
        ts = {"bf16": torch.randn(257, 33, device="cuda", generator=g).to(torch.bfloat16),
              "fp32": torch.randn(1000, device="cuda", generator=g),
              "int8": torch.randint(-128, 128, (64, 7, 3), dtype=torch.int8, device="cuda", generator=g),
              "wide": torch.randn(9, 8192, device="cuda", generator=g)}
        store.batch_put(list(ts), list(ts.values()))
        cases = [("bf16", 0, 257), ("bf16", 100, 101), ("bf16", 3, 200), ("fp32", 999, 1000), ("fp32", 10, 10), ("int8", 5, 63),
                 ("wide", 1, 8), ("wide", 4, 5)]
        for k, a, b in cases:
            got = store.get_rows(k, a, b)
            assert got.dtype == ts[k].dtype and got.shape == ts[k][a:b].shape and torch.equal(got, ts[k][a:b]), (k, a, b)
        outs = store.batch_get_rows([k for k, _, _ in cases], [a for _, a, _ in cases], [b for _, _, b in cases])
        assert all(torch.equal(o, ts[k][a:b]) for o, (k, a, b) in zip(outs, cases))
        for a, b in ((-1, 3), (5, 4), (0, 258)):
            with pytest.raises(IndexError):
                store.get_rows("bf16", a, b)
        store.put("scalar", torch.tensor(3.0, device="cuda"))
        with pytest.raises(IndexError):
            store.get_rows("scalar", 0, 0)
        # MXFP8-packed: read whole, unpacked and sliced
        x = torch.randn(96, 64, device="cuda", generator=g).to(torch.bfloat16)
        store.put("packed", x, pack_fp8=True)
        whole = store.get("packed")
        assert torch.equal(store.get_rows("packed", 10, 50), whole[10:50])
    finally:
        cl.stop()
