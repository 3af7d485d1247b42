"""Strided device gets on the GPU: the strided store window of bb_xfer (XFER_STRIDED) through XferEngine, the client's
batch_get_device_strided on a GpuRankCluster, and TensorStore.get_slice, against numpy / torch slices and the CPU digest
models.  A strided descriptor reads and hashes its whole object and stores only its rows, densely, so every check covers
the stored bytes, the guard bytes on both sides of every result, the digest and the verify status."""
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


def stored(n, w):
    """(object offsets, result offsets) of the bytes a window stores: w = None (whole), (lo, hi) or (lo, hi, pitch, width,
    phase); result offsets are relative to dst[0]."""
    if w is None:
        x = np.arange(n, dtype=np.int64)
        return x, x
    x = np.arange(w[0], w[1], dtype=np.int64)
    if len(w) == 2:
        return x, x
    pitch, width, phase = w[2:]
    y = x + phase
    keep = y % pitch < width
    return x[keep], (y // pitch * width + y % pitch)[keep]


class Batch:
    """Items reading objects of `src` (object i at src_offs[i], n[i] bytes) into one guard-filled destination buffer, each
    at its own region with guard bytes on both sides; dst[0] of a strided item is placed so that its rows are co-aligned
    (unless `skew` moves it)."""

    def __init__(self, bb, src, src_offs, sizes, wins, algo, verify=True, expect=None, skew=0):
        self.bb, self.src, self.src_offs, self.sizes, self.wins = bb, src, src_offs, sizes, wins
        self.maps, self.bases, o = [], [], 64
        for n, w in zip(sizes, wins):
            xs, ds = stored(n, w)
            lo_d = int(ds.min()) if ds.size else 0
            hi_d = int(ds.max()) + 1 if ds.size else 0
            # region start o holds result offset lo_d, so dst[0] = o - lo_d: the engine wants dst[0] 16-byte aligned, and for
            # a strided window dst[0] + phase - r_lo * (pitch - width)
            res = lo_d
            if w is not None and len(w) == 5:
                pitch, width, phase = w[2:]
                res = lo_d - phase + (w[0] + phase) // pitch * (pitch - width)
            o = (o + 15) // 16 * 16 + res % 16 + skew
            self.bases.append(o - lo_d)
            self.maps.append((xs, ds))
            o += hi_d - lo_d + 64
        self.dst = torch.full((o + 64,), GUARD, dtype=torch.uint8, device="cuda")
        model = _model(bb, algo)
        host = src.cpu().numpy()
        self.digests = [model(host[so:so + n]) for so, n in zip(src_offs, sizes)] if expect is None else expect
        self.items = []
        for so, n, w, b, d in zip(src_offs, sizes, wins, self.bases, self.digests):
            flags = bb.XFER_VERIFY if (verify and algo != "NONE") else 0
            it = (src.data_ptr() + so, self.dst.data_ptr() + b, n, d, flags)
            self.items.append(it if w is None else it + (0, w))

    def want(self):
        want = np.full(self.dst.numel(), GUARD, dtype=np.uint8)
        host = self.src.cpu().numpy()
        for so, b, (xs, ds) in zip(self.src_offs, self.bases, self.maps):
            want[b + ds] = host[so + xs]
        return torch.from_numpy(want).cuda()

    def check(self, what):
        torch.cuda.synchronize()
        want = self.want()
        if not torch.equal(self.dst, want):
            bad = (self.dst != want).nonzero().flatten()[:8].tolist()
            pytest.fail(f"{what}: bytes differ at {bad}; bases {self.bases[:8]}")


def patterns(n):
    """Strided windows (lo, hi, pitch, width, phase) of an n-byte object: pitches below, equal to and above 16 KiB; widths
    of 1, 15, 16 and 17 bytes and width == pitch; phases 0, 5 and pitch - 1; windows that start and end inside a row; rows
    that straddle tile edges."""
    out = []
    for pitch0 in (992, T, 40000):
        for width in (1, 15, 16, 17, None):
            pitch = pitch0 + (width % 16 if width else 0)  # multi-row windows need (pitch - width) % 16 == 0
            wd = width or pitch
            for phase in (0, 5, pitch - 1):
                out.append((0, n, pitch, wd, phase))
            out.append((T - 3, n - 7, pitch, wd, 11))
    out.append((5 * T + 100, 5 * T + 100, 992, 16, 0))   # empty
    out.append((T - 8, T + 8, 100, 16, 24))              # one row across a tile edge
    return out


@pytest.mark.parametrize("algo", ALGOS)
def test_strided_windows_at_every_grid(bb, eng, algo):
    """Every pattern of a 8-tile object, one device-table batch (more than 8 items, whole and windowed items mixed in),
    at grids of 1, 7, the SM count and twice the SM count, so that rows straddle tile edges and CTA runs."""
    A = getattr(bb.ChecksumAlgo, algo)
    n = 8 * T + 77
    src = _random(bb, n, 17)
    ps = patterns(n)
    for chunk in range(0, len(ps), 12):
        ws = ps[chunk:chunk + 12] + [None, (T + 1, 3 * T - 1)]
        b = Batch(bb, src, [0] * len(ws), [n] * len(ws), ws, algo)
        for g in GRIDS:
            eng.set_max_ctas(_grid(g))
            b.dst.fill_(GUARD)
            dg, st, _ = eng.run(b.items, A, _stream())
            assert st == [0] * len(ws), (g, st)
            if algo != "NONE":
                assert dg == b.digests, g
            b.check(f"{algo} chunk={chunk} grid={g}")


@pytest.mark.parametrize("algo", ALGOS)
def test_inline_batches_mix_strided_windowed_and_whole(bb, eng, algo):
    """Batches of <= 8 descriptors carry their row patterns in the kernel parameters; digests and status equal those of a
    plain verified get of the same objects."""
    A = getattr(bb.ChecksumAlgo, algo)
    sizes = [3 * T + 7, 5000, 2 * T + 1, 100, 4 * T]
    offs = [0, 65536, 131072, 196608, 262144]
    src = _random(bb, 400000, 7)
    wins = [(0, 3 * T + 7, 256, 128, 0), None, (1, 2 * T, 4097, 1, 7), (8, 100, 40, 24, 39), (T - 1, 4 * T, 6000, 6000, 5)]
    b = Batch(bb, src, offs, sizes, wins, algo)
    dg, st, _ = eng.run(b.items, A, _stream())
    b.check("inline")
    plain = Batch(bb, src, offs, sizes, [None] * 5, algo)
    pdg, pst, _ = eng.run(plain.items, A, _stream())
    assert st == pst == [0] * 5 and dg == pdg


@pytest.mark.parametrize("algo", ALGOS)
def test_a_flipped_byte_outside_the_pattern_fails_verification(bb, eng, algo):
    A = getattr(bb.ChecksumAlgo, algo)
    n = 3 * T + 7
    src = _random(bb, n, 3)
    good = _model(bb, algo)(src.cpu().numpy())
    src[300] ^= 0xFF  # in the gap of every pattern below
    for w in [(0, n, 256, 32, 0), (200, 2 * T, 1008, 16, 900), (T, n, 64, 16, 0)]:
        b = Batch(bb, src, [0], [n], [w], algo, expect=[good])
        _, st, _ = eng.run(b.items, A, _stream())
        assert st == [0 if algo == "NONE" else 1], (w, st)
        b.check("the rows are stored even when the object fails verification")


def test_none_reads_only_the_trimmed_span(bb, eng):
    """Without a checksum a strided descriptor is trimmed to [lo & ~15, hi) like a plain window, with its phase and base
    moved so that the same bytes land at the same addresses."""
    n = 10 * T + 5
    src = _random(bb, n, 9)
    wins = [(5 * T + 3, 7 * T + 40, 1000, 40, 3), (3 * T + 17, n, T + 16, 16, T), (9 * T + 1, n, 33, 1, 32)]
    b = Batch(bb, src, [0] * len(wins), [n] * len(wins), wins, "NONE")
    eng.set_tile_trace(True)
    _, st, _ = eng.run(b.items, bb.ChecksumAlgo.NONE, _stream())
    tiles = sum(-(-(w[1] - (w[0] & ~15)) // T) for w in wins)
    assert st == [0] * len(wins) and len(eng.tile_trace()) == 4 * tiles
    b.check("trimmed")


def test_strided_items_take_the_fused_kernel(bb, eng):
    src = _random(bb, 8 * 4096, 5)
    b = Batch(bb, src, [0, 4096], [4096, 100], [(0, 4096, 64, 16, 0), (0, 100, 20, 4, 0)], "XXH3")
    sl, mb, la = eng.small_launches, eng.mailbox_requests, eng.launches
    _, st, _ = eng.run(b.items, bb.ChecksumAlgo.XXH3, _stream())
    assert st == [0] * 2 and eng.small_launches == sl and eng.mailbox_requests == mb and eng.launches == la + 1
    b.check("small")


def test_rejected_patterns(bb, eng):
    src = _random(bb, 2 * T, 1)
    dst = torch.full((2 * T,), GUARD, dtype=torch.uint8, device="cuda")
    s, d = src.data_ptr(), dst.data_ptr()
    A = bb.ChecksumAlgo.XXH3
    bad = [((s, d, 1000, 0, 0, 0, (0, 1000, 100, 0, 0)), "INVALID_ARGUMENT"),        # width 0
           ((s, d, 1000, 0, 0, 0, (0, 1000, 100, 101, 0)), "INVALID_ARGUMENT"),      # width > pitch
           ((s, d, 1000, 0, 0, 0, (0, 1000, 100, 50, 100)), "INVALID_ARGUMENT"),     # phase >= pitch
           ((s, d, 1000, 0, 0, 0, (0, 1001, 100, 50, 0)), "INVALID_ARGUMENT"),       # past the object
           ((s, d, 1000, 0, bb.XFER_STRIDED), "INVALID_ARGUMENT"),                   # strided without a window
           ((s, d, 1000, 0, 0, 0, (0, 1000, 100, 52, 4)), "INVALID_ADDRESS"),        # dst[0] + phase misaligned
           ((s, d, 1000, 0, 0, 0, (0, 1000, 100, 60, 0)), "INVALID_ADDRESS"),        # gap of 40 bytes
           ((s, d + 8, 1000, 0, 0, 0, (0, 1000, 96, 80, 0)), "INVALID_ADDRESS")]     # dst[0] misaligned
    for it, err in bad:
        with pytest.raises(RuntimeError, match=err):
            eng.run([it], A, _stream())
    # a window inside one row may leave any gap: that row's base is what has to be co-aligned.  Bytes [130, 160) of row 1
    # land at dst[0] + 60 + 30, which is d + 18 (congruent to 130 mod 16) for dst[0] = d - 72.
    eng.run([(s, d - 72, 1000, 0, 0, 0, (130, 180, 100, 60, 0))], bb.ChecksumAlgo.NONE, _stream())
    torch.cuda.synchronize()
    assert torch.equal(dst[18:48], src[130:160]) and bool((dst[:18] == GUARD).all()) and bool((dst[48:] == GUARD).all())


# ---------------------------------------------------------------------------------------------------- client


def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


def _fabric_get_bytes(client):
    return sum(int(line.split()[1]) for line in client.metrics_text().splitlines()
               if line.startswith('bb_fabric_bytes_total{') and 'dir="get"' in line)


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


def _strided_get(cl, keys, pats, skew=None):
    """Strided gets into one guard-filled device buffer, each result at a region congruent to its offset mod 16 (+ skew);
    returns (error codes, buffer, region offsets)."""
    regions, o = [], 256
    for i, (off, w, _, r) in enumerate(pats):
        regions.append(o + off % 16 + (skew or {}).get(i, 0))
        o += (w * r + 255) // 256 * 256 + 256
    out = torch.full((o,), GUARD, dtype=torch.uint8, device="cuda")
    ecs = cl.client.batch_get_device_strided(keys, [out.data_ptr() + r for r in regions], [p[0] for p in pats], [p[1] for p in pats],
                                             [p[2] for p in pats], [p[3] for p in pats], _stream())
    return ecs, out, regions


def _check_strided(out, regions, objs, pats, ok):
    want = torch.full_like(out, GUARD)
    for r, obj, (off, w, p, n), good in zip(regions, objs, pats, ok):
        if good and w and n:
            want[r:r + w * n] = obj[off:off + (n - 1) * p + w].unfold(0, w, p).reshape(-1) if n > 1 else obj[off:off + w]
    torch.cuda.synchronize()
    if not torch.equal(out, want):
        pytest.fail(f"strided get wrote wrong bytes at {(out != want).nonzero().flatten()[:8].tolist()}")


@pytest.mark.parametrize("algo", ["XXH3", "CRC32C", "BBH64"])
def test_client_strided_fails_over_from_a_copy_corrupt_in_a_gap(bb, algo):
    """Replication 1 and 2 on one slab (the client reads copy 0 first: every copy is local).  Copy 0 is corrupt in a gap
    between rows: the rows come from the replica after one fail-over; with one copy the get fails."""
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=128 << 20, cluster_id=f"t-str-rep-{algo}", max_replicas=3)
    try:
        n = 3 * T + 7
        src = _random(bb, n, 21)
        for rep in (1, 2):
            key = f"s{rep}"
            assert cl.client.batch_put_device([key], [src.data_ptr()], [n], _cfg(bb, algo, rep), _stream()) == [bb.ErrorCode.OK]
            _flip(bb, cl, cl.client.get_workers(key)[0].shards[0], 16 + 200)
            pat = (16, 128, 1024, 40)  # byte 216 lies in the gap after row 0
            mm, l0 = _counter(cl.client, "checksum_mismatch_total"), cl.fabric.launches
            ecs, out, regions = _strided_get(cl, [key], [pat])
            ok = rep > 1
            assert ecs == [bb.ErrorCode.OK if ok else bb.ErrorCode.CHECKSUM_MISMATCH], (rep, ecs)
            assert _counter(cl.client, "checksum_mismatch_total") > mm
            if ok:
                _check_strided(out, regions, [src], [pat], [True])
                assert cl.fabric.launches == l0 + 2
    finally:
        cl.stop()


@pytest.mark.parametrize("algo", ALGOS)
def test_client_strided_over_hbm_and_dram_in_one_launch(bb, algo):
    """Objects in HBM and in a pinned DRAM pool, and objects striped over both (rows across the shard edge): one batch of
    strided gets costs one launch; a misaligned item is staged alone; errors fail alone; one row equals the range get."""
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id=f"t-str-tier-{algo}", dram_bytes=64 << 20)
    try:
        sizes = [5 * T + 11, 70001, 2 * MiB + 5, 2 * MiB]
        srcs = [_random(bb, n, 30 + i) for i, n in enumerate(sizes)]
        keys = []
        for i, (n, s) in enumerate(zip(sizes, srcs)):
            for tier in ("RAM_GPU", "RAM_CPU"):
                k = f"{tier}/{i}"
                assert cl.client.batch_put_device([k], [s.data_ptr()], [n], _cfg(bb, algo, 1, tier), _stream()) == [bb.ErrorCode.OK]
                keys.append((k, i))
        striped = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=2, ttl_ms=0, min_shard_size=4096,
                                  checksum=getattr(bb.ChecksumAlgo, algo), preferred_classes=[bb.StorageClass.RAM_GPU, bb.StorageClass.RAM_CPU])
        assert cl.client.batch_put_device(["striped"], [srcs[3].data_ptr()], [sizes[3]], striped, _stream()) == [bb.ErrorCode.OK]
        shards = cl.client.get_workers("striped")[0].shards
        assert len(shards) == 2 and shards[0].length % 16 == 0, [s.length for s in shards]
        keys.append(("striped", 3))
        ks, objs, pats = [], [], []
        for k, i in keys:
            n = sizes[i]
            for p in [(16, 96, 1024, (n - 112) // 1024), (5, 1, 17, 2000), (T - 16, 48, T, (n - T - 32) // T), (32, 0, 64, 9),
                      (0, 64, 64, n // 64)]:
                ks.append(k), objs.append(srcs[i]), pats.append(p)
        l0, st0 = cl.fabric.launches, _counter(cl.client, "device_get_host_staged_total")
        ecs, out, regions = _strided_get(cl, ks, pats)
        assert ecs == [bb.ErrorCode.OK] * len(ks), ecs
        assert cl.fabric.launches == l0 + 1 and _counter(cl.client, "device_get_host_staged_total") == st0
        _check_strided(out, regions, objs, pats, [True] * len(ks))
        # one item with a misaligned virtual base and one with a 40-byte gap go through the host; the rest keep one launch
        pats2 = [(16, 96, 1024, 40), (16, 96, 1024, 40), (0, 24, 64, 100), (48, 16, 32, 1000)]
        l0, st0 = cl.fabric.launches, _counter(cl.client, "device_get_host_staged_total")
        ecs, out, regions = _strided_get(cl, [keys[0][0]] * 4, pats2, {1: 3})
        assert ecs == [bb.ErrorCode.OK] * 4
        assert cl.fabric.launches == l0 + 1 and _counter(cl.client, "device_get_host_staged_total") == st0 + 2
        _check_strided(out, regions, [srcs[0]] * 4, pats2, [True] * 4)
        E = bb.ErrorCode
        ecs, out, regions = _strided_get(cl, [keys[0][0], "missing", keys[1][0], keys[2][0]],
                                         [(0, 65, 64, 2), (0, 16, 32, 2), (48, 64, 80, 3), (16, 16, 2**63, 3)])
        assert ecs == [E.INVALID_ARGUMENT, E.OBJECT_NOT_FOUND, E.OK, E.VALUE_OUT_OF_RANGE], ecs
        # rows == 1: the same bytes counted and the same launches as the range get
        b0, l0 = _fabric_get_bytes(cl.client), cl.fabric.launches
        ecs, out, regions = _strided_get(cl, ["striped"], [(MiB - 40, 100, 7, 1)])
        assert ecs == [E.OK]
        _check_strided(out, regions, [srcs[3]], [(MiB - 40, 100, 7, 1)], [True])
        b1, l1 = _fabric_get_bytes(cl.client), cl.fabric.launches
        rng = torch.full((256,), GUARD, dtype=torch.uint8, device="cuda")
        assert cl.client.batch_get_device_range(["striped"], [rng.data_ptr() + (MiB - 40) % 16], [MiB - 40], [100], _stream()) == [E.OK]
        assert _fabric_get_bytes(cl.client) - b1 == b1 - b0 and cl.fabric.launches - l1 == l1 - l0 == 1
        # rows only in the second shard: the first is not read (without a checksum only the rows' aligned span is)
        b0 = _fabric_get_bytes(cl.client)
        pat = (shards[0].length + 32, 16, 64, 100)
        ecs, out, regions = _strided_get(cl, ["striped"], [pat])
        assert ecs == [E.OK]
        _check_strided(out, regions, [srcs[3]], [pat], [True])
        assert _fabric_get_bytes(cl.client) - b0 == (shards[1].length if algo != "NONE" else 99 * 64 + 16)
    finally:
        cl.stop()


# ---------------------------------------------------------------------------------------------------- TensorStore


def test_tensor_store_get_slice(bb):
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id="t-str-slice")
    try:
        store = TensorStore(cl.client)
        g = torch.Generator(device="cuda").manual_seed(5)
        ts = {}
        for dt in (torch.uint8, torch.bfloat16, torch.float32, torch.int64):
            for shape in ((37,), (9, 33), (5, 6, 7), (3, 4, 5, 16)):
                x = torch.randint(0, 255, shape, dtype=torch.int64, device="cuda", generator=g)
                ts[f"{dt}/{len(shape)}"] = x.to(dt) if dt != torch.bfloat16 else torch.randn(shape, device="cuda", generator=g).to(dt)
        store.batch_put(list(ts), list(ts.values()))
        cases = []
        for k, t in ts.items():
            for d in range(-t.dim(), t.dim()):
                n = t.shape[d]
                for a, b in ((0, n), (1, n - 1), (n // 2, n // 2), (n - 1, n), (0, 1)):
                    cases.append((k, d, a, b))
        for k, d, a, b in cases:
            got = store.get_slice(k, d, a, b)
            want = ts[k].narrow(d, a, b - a).contiguous()
            assert got.dtype == want.dtype and got.shape == want.shape and got.is_contiguous(), (k, d, a, b)
            assert torch.equal(got, want), (k, d, a, b)
        outs = store.batch_get_slices([c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases])
        assert all(torch.equal(o, ts[k].narrow(d, a, b - a)) for o, (k, d, a, b) in zip(outs, cases))
        for d, a, b in ((2, 0, 1), (-3, 0, 1), (1, -1, 3), (1, 5, 4), (1, 0, 34)):
            with pytest.raises(IndexError):
                store.get_slice("torch.float32/2", d, a, b)
        store.put("scalar", torch.tensor(3.0, device="cuda"))
        with pytest.raises(IndexError):
            store.get_slice("scalar", 0, 0, 0)
        # MXFP8-packed: whole fused get, then narrowed
        x = torch.randn(96, 64, device="cuda", generator=g).to(torch.bfloat16)
        store.put("packed", x, pack_fp8=True)
        whole = store.get("packed")
        assert torch.equal(store.get_slice("packed", 1, 10, 50).view(torch.int16), whole[:, 10:50].contiguous().view(torch.int16))
        assert torch.equal(store.get_slice("packed", 0, 10, 50).view(torch.int16), whole[10:50].view(torch.int16))
    finally:
        cl.stop()
