"""Gets into strided destinations on the GPU: the scattering store of bb_xfer and of the fused MXFP8 unpack (XFER_SCATTER)
through XferEngine, the client's batch_get_device_scatter / batch_get_device_fp8_scatter on a GpuRankCluster, and
TensorStore.get_into of sliced tensors.  A scattered descriptor stores its object's bytes into rows of a strided destination;
the tile in shared memory is the object's own, so every check covers the stored rows, the guard bytes around and between
them, and the digest, which must equal that of a plain get of the same object."""
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


def rows_index(n, pitch, width, phase):
    """Offset (from the pattern's row 0) of each object byte: the rule of SourceRows, on either side."""
    y = np.arange(n, dtype=np.int64) + phase
    return y // width * pitch + y % width


class Batch:
    """One launch mixing scattered gets with plain, windowed, strided-window and gathered items.  Every object comes from
    one random source buffer, every destination is a region of one guard-filled buffer.  A spec is (kind, nbytes, arg):
    scatter (pitch, width, phase) | plain None | window (lo, hi) | swin (pitch, width) | gather (pitch, width, phase)."""

    def __init__(self, bb, specs, algo, seed=11):
        self.bb, self.specs, self.algo = bb, specs, algo
        src_at, o, objs_idx = [], 64, []
        for kind, n, arg in specs:
            ix = rows_index(n, *arg) if kind == "gather" else np.arange(n, dtype=np.int64)
            o = (o + 15) // 16 * 16 + ((16 - arg[2] % 16) % 16 if kind == "gather" else 0)
            src_at.append(o)
            objs_idx.append(ix)
            o += (int(ix.max()) + 1 if n else 0) + 64
        self.src = _random(bb, o + 64, seed)
        host = self.src.cpu().numpy()
        self.objs = [host[s + ix] for s, ix in zip(src_at, objs_idx)]
        model = _model(bb, algo)
        self.digests = [model(b.tobytes()) for b in self.objs]
        # destinations: the region of item i and where each of its stored bytes lands in it
        self.places, self.regions, o = [], [], 64
        for (kind, n, arg), obj in zip(specs, self.objs):
            if kind == "scatter":
                pitch, width, phase = arg
                o = (o + 15) // 16 * 16 + (16 - phase % 16) % 16
                at, stored = rows_index(n, pitch, width, phase), np.arange(n)
            elif kind == "window":
                o = (o + 15) // 16 * 16 + arg[0] % 16
                at, stored = np.arange(arg[1] - arg[0]), np.arange(arg[0], arg[1])
            elif kind == "swin":
                pitch, width = arg
                o = (o + 15) // 16 * 16
                x = np.arange(n)
                stored = x[x % pitch < width]
                at = stored // pitch * width + stored % pitch
            else:
                o = (o + 15) // 16 * 16
                at, stored = np.arange(n), np.arange(n)
            self.regions.append(o)
            self.places.append((o + at, stored))
            o += (int(at.max()) + 1 if at.size else 0) + 64
        self.dst = torch.full((o + 64,), GUARD, dtype=torch.uint8, device="cuda")
        verify = 0 if algo == "NONE" else bb.XFER_VERIFY
        self.items = []
        for (kind, n, arg), s, r, dg in zip(specs, src_at, self.regions, self.digests):
            sp, dp = self.src.data_ptr() + s, self.dst.data_ptr() + r
            if kind == "scatter":
                it = (sp, dp, n, dg, verify, 0, None, None, arg)
            elif kind == "window":
                it = (sp, dp - arg[0], n, dg, verify, 0, arg)
            elif kind == "swin":
                it = (sp, dp, n, dg, verify, 0, (0, n, arg[0], arg[1], 0))
            elif kind == "gather":
                it = (sp, dp, n, dg, verify, 0, None, arg)
            else:
                it = (sp, dp, n, dg, verify)
            self.items.append(it)

    def want(self):
        w = np.full(self.dst.numel(), GUARD, dtype=np.uint8)
        for obj, (at, stored) in zip(self.objs, self.places):
            w[at] = obj[stored]
        return w

    def check(self, what):
        torch.cuda.synchronize()
        got, want = self.dst.cpu().numpy(), self.want()
        if not np.array_equal(got, want):
            pytest.fail(f"{what}: bytes differ at {np.nonzero(got != want)[0][:8].tolist()}")


def scatter_specs():
    """Widths from 1 byte to more than a tile, rows spanning tiles, thousands of rows per tile at width 16 / pitch 32,
    phases with head and tail bytes in every row, objects of 1 byte to several MiB."""
    return [("scatter", 1, (17, 1, 0)), ("scatter", 3000, (32, 16, 0)), ("scatter", 3 * T + 5, (32, 16, 0)),
            ("scatter", 5000, (33, 17, 16)), ("scatter", 2 * T + 5, (4016, 4000, 123)), ("scatter", 3 * T + 77, (T + 48, T + 16, 7)),
            ("scatter", 2 * T, (2 * T + 35, T + 3, T)), ("scatter", 4 * MiB + 3, (144, 128, 0)),
            ("scatter", 6 * T + 11, (4096 + 16, 4096, 4000))]


@pytest.mark.parametrize("algo", ALGOS)
def test_scattered_gets_at_every_grid(bb, eng, algo):
    """Every pattern in one device-table batch with plain, windowed, strided-window and gathered items mixed in, at grids
    of 1, 7, the SM count and twice the SM count: the rows equal the object, every guard byte is intact, the digests equal
    the CPU model, and a wrong expected digest gives status 1."""
    A = getattr(bb.ChecksumAlgo, algo)
    specs = scatter_specs() + [("plain", 3 * T + 7, None), ("window", 2 * T + 9, (100, T + 333)), ("swin", 5 * T, (4096, 2048)),
                               ("gather", 2 * T + 1, (48, 32, 5))]
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
    if algo != "NONE":
        bad = [it[:3] + (it[3] ^ 1,) + it[4:] if k == "scatter" else it for it, (k, _, _) in zip(b.items, specs)]
        _, st, _ = eng.run(bad, A, _stream())
        assert st == [1 if k == "scatter" else 0 for k, _, _ in specs]


@pytest.mark.parametrize("algo", ALGOS)
def test_inline_batches_mix_scattered_and_plain(bb, eng, algo):
    """Batches of <= 8 descriptors carry their destination rows in the kernel parameters."""
    A = getattr(bb.ChecksumAlgo, algo)
    specs = [("scatter", 3 * T + 7, (256, 128, 0)), ("plain", 5000, None), ("scatter", 2 * T + 1, (4113, 1, 0)),
             ("scatter", 100, (40, 24, 13)), ("gather", 4 * T, (6000, 6000 - 16 * 7, 5)), ("window", T, (7, 9000))]
    for g in GRIDS:
        eng.set_max_ctas(_grid(g))
        b = Batch(bb, specs, algo, seed=3)
        dg, st, _ = eng.run(b.items, A, _stream())
        assert st == [0] * len(specs)
        if algo != "NONE":
            assert dg == b.digests
        b.check(f"inline {algo} grid={g}")


def test_small_scattered_items_take_the_fused_kernel_and_occupancy_holds(bb, eng):
    """Objects of 4 KiB and less, scattered, never take the warp-per-object kernel or the mailbox; the fused kernel keeps
    two resident CTAs per SM (one for CRC32C)."""
    b = Batch(bb, [("scatter", 4096, (64, 16, 0)), ("scatter", 100, (20, 4, 0)), ("scatter", 1, (17, 1, 0))], "XXH3")
    sl, mb, la = eng.small_launches, eng.mailbox_requests, eng.launches
    dg, st, _ = eng.run(b.items, bb.ChecksumAlgo.XXH3, _stream())
    assert st == [0] * 3 and dg == b.digests
    assert eng.small_launches == sl and eng.mailbox_requests == mb and eng.launches == la + 1
    b.check("small")
    for algo in ALGOS:
        want = 1 if algo == "CRC32C" else 2
        assert bb.xfer_geometry(getattr(bb.ChecksumAlgo, algo), 10000)["resident_ctas_per_sm"] == want, algo


def test_rejected_scatters(bb, eng):
    src = _random(bb, 4 * T, 1)
    dst = torch.full((2 * T,), GUARD, dtype=torch.uint8, device="cuda")
    s, d = src.data_ptr(), dst.data_ptr()
    A = bb.ChecksumAlgo.XXH3
    pat = (96, 80, 0)
    bad = [((s, d, 1000, 0, 0, 0, None, None, (100, 0, 0)), "INVALID_ARGUMENT"),            # width 0
           ((s, d, 1000, 0, 0, 0, None, None, (100, 101, 0)), "INVALID_ARGUMENT"),          # width > pitch
           ((s, d, 1000, 0, 0, 0, None, None, (100, 50, 50)), "INVALID_ARGUMENT"),          # phase >= width
           ((s, d, 1000, 0, bb.XFER_SCATTER), "INVALID_ARGUMENT"),                           # flag without a pattern
           ((s, d, 1000, 0, 0, 0, (0, 500), None, pat), "INVALID_ARGUMENT"),                 # with a window
           ((s, d, 1000, 0, 0, 0, (0, 1000, 96, 80, 0), None, pat), "INVALID_ARGUMENT"),     # with a strided window
           ((s, d, 1000, 0, 0, 0, None, pat, pat), "INVALID_ARGUMENT"),                      # with a gather pattern
           ((s, [], 1000, 0, bb.XFER_RAW_SUM, 0, None, None, pat), "INVALID_ARGUMENT"),      # with RAW_SUM
           ((s, d, 1008, 0, bb.XFER_MULTIMEM, 0, None, None, pat), "INVALID_ARGUMENT"),      # with MULTIMEM
           ((s, [d, d + T], 1000, 0, 0, 0, None, None, pat), "INVALID_ARGUMENT"),            # two destinations
           ((s, d, 1000, 0, 0, 0, None, None, (96, 80, 5)), "INVALID_ADDRESS"),              # dst + phase misaligned
           ((s, d + 8, 1000, 0, 0, 0, None, None, pat), "INVALID_ADDRESS"),                  # dst misaligned
           ((s, d, 1000, 0, 0, 0, None, None, (100, 60, 0)), "INVALID_ADDRESS"),             # gap of 40 bytes
           ((s + 8, d, 1000, 0, 0, 0, None, None, pat), "INVALID_ADDRESS")]                  # src misaligned
    for it, err in bad:
        with pytest.raises(RuntimeError, match=err):
            eng.run([it], A, _stream())
    torch.cuda.synchronize()
    assert bool((dst == GUARD).all())
    # an object inside one row may have any gap: only dst + phase has to be aligned
    eng.run([(s, d - 4, 50, 0, 0, 0, None, None, (100, 60, 4))], A, _stream())
    torch.cuda.synchronize()
    assert torch.equal(dst[:50], src[:50]) and bool((dst[50:] == GUARD).all())


# ---------------------------------------------------------------------------------------------------- fused MXFP8 unpack


def _bf16(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(n, device="cuda", generator=g) * 3).to(torch.bfloat16)


def test_fused_unpack_scatters_bit_exact(bb, eng):
    """Packed objects unpacked into 2-row and many-row patterns, with tail tiles and phases: bit-exact against mxfp8_unpack
    of the same packed bytes scattered in numpy, guards intact, the digest that of a plain unpack, and a wrong expected
    digest gives status 1."""
    # (n_elems, (pitch, width, phase) in elements)
    specs = [(2 * T, (T + 8, T, 0)), (3 * T + 96, (40, 32, 0)), (T + 32, (2 * T + 40, 2 * T, 5)), (64, (24, 16, 8)),
             (8 * T, (4096 + 64, 4096, 1000)), (T * 2 + 32 * 7, (3 * T + 16, T + 8, 0))]
    packed, wides, refs = [], [], []
    for k, (n, _) in enumerate(specs):
        w = _bf16(n, k)
        p = torch.empty(n + n // 32, dtype=torch.uint8, device="cuda")
        bb.mxfp8_pack(w.data_ptr(), n, p.data_ptr(), _stream())
        r = torch.empty(n, dtype=torch.bfloat16, device="cuda")
        bb.mxfp8_unpack(p.data_ptr(), n, r.data_ptr(), _stream())
        packed.append(p), wides.append(w), refs.append(r.view(torch.int16).cpu().numpy())
    plain_out = [torch.empty(n, dtype=torch.bfloat16, device="cuda") for n, _ in specs]
    pdg, pst, _ = eng.run_fp8([(o.data_ptr(), p.data_ptr(), n) for o, p, (n, _) in zip(plain_out, packed, specs)], True, _stream())
    assert pst == [0] * len(specs)
    regions, o = [], 64
    for n, (pitch, width, phase) in specs:
        o = (o + 7) // 8 * 8 + (8 - phase % 8) % 8  # dst + 2 * phase 16-byte aligned
        regions.append(o)
        o += int(rows_index(n, pitch, width, phase).max()) + 64
    dst = torch.full((o + 64,), -0x5A5B, dtype=torch.int16, device="cuda")
    items = [(dst.data_ptr() + 2 * r, p.data_ptr(), n, dg, None, None, pat) for r, p, (n, pat), dg in zip(regions, packed, specs, pdg)]
    for g in (1, "sms"):
        eng.set_max_ctas(_grid(g))
        dst.fill_(-0x5A5B)
        dg, st, _ = eng.run_fp8(items, True, _stream())
        assert st == [0] * len(specs) and dg == pdg, g
        torch.cuda.synchronize()
        want = np.full(dst.numel(), -0x5A5B, dtype=np.int16)
        for r, ref, (n, pat) in zip(regions, refs, specs):
            want[r + rows_index(n, *pat)] = ref
        got = dst.cpu().numpy()
        assert np.array_equal(got, want), (g, np.nonzero(got != want)[0][:8])
    eng.set_max_ctas(0)
    bad = [it[:3] + (it[3] ^ 1,) + it[4:] for it in items]
    _, st, _ = eng.run_fp8(bad, True, _stream())
    assert st == [1] * len(specs)
    # a scatter pattern on a pack, or with a window, is refused
    w = wides[0]
    with pytest.raises(RuntimeError, match="INVALID_ARGUMENT"):
        eng.run_fp8([(w.data_ptr(), packed[0].data_ptr(), 2 * T, None, None, None, (T + 8, T, 0))], False, _stream())
    with pytest.raises(RuntimeError, match="INVALID_ARGUMENT"):
        eng.run_fp8([(dst.data_ptr(), packed[0].data_ptr(), 2 * T, None, (0, T), None, (T + 8, T, 0))], True, _stream())
    with pytest.raises(RuntimeError, match="INVALID_ADDRESS"):
        eng.run_fp8([(dst.data_ptr() + 2, packed[0].data_ptr(), 2 * T, None, None, None, (T + 8, T, 0))], True, _stream())


# ---------------------------------------------------------------------------------------------------- client


def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


@pytest.mark.parametrize("algo", ALGOS)
def test_client_scattered_gets(bb, algo):
    """Objects in HBM, replicated, in a pinned DRAM pool, and striped over both (shard edges mid-row): one call scatters
    every fused item in one launch; misaligned pointers and odd gaps are staged alone; no byte outside the rows changes."""
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=128 << 20, cluster_id=f"t-scat-{algo}", dram_bytes=64 << 20, max_replicas=3)
    try:
        A = getattr(bb.ChecksumAlgo, algo)
        striped = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=2, ttl_ms=0, min_shard_size=4096, checksum=A,
                                  preferred_classes=[bb.StorageClass.RAM_GPU, bb.StorageClass.RAM_CPU])
        plain = bb.WorkerConfig(replication_factor=2, max_workers_per_copy=1, ttl_ms=0, checksum=A, preferred_classes=[bb.StorageClass.RAM_GPU])
        dram = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, checksum=A, preferred_classes=[bb.StorageClass.RAM_CPU])
        sizes = [96 * 21845, 300000, 3 * T + 5, 1000]
        cfgs = [striped, plain, dram, plain]
        objs = []
        for k, (n, cfg) in enumerate(zip(sizes, cfgs)):
            t = _random(bb, n, 50 + k)
            assert cl.client.batch_put_device([f"o{k}"], [t.data_ptr()], [n], cfg, _stream()) == [bb.ErrorCode.OK]
            objs.append(t.cpu().numpy()[:n])
        # (key, width, pitch, rows, skew)
        items = [(0, 96, 128, 21845, 0), (1, 1000, 1048, 300, 0), (2, T, T + 48, 4, 0), (3, 16, 48, 63, 0),
                 (1, 1000, 1048, 300, 3), (1, 1000, 1033, 300, 0), (2, 3 * T + 5, 3 * T + 5, 1, 0)]
        regions, o = [], 64
        for _, w, p, r, sk in items:
            regions.append(o + sk)
            o = (o + sk + (r - 1) * p + w + 15) // 16 * 16 + 64
        for rep in range(2):
            dst = torch.full((o + 64,), GUARD, dtype=torch.uint8, device="cuda")
            l0, st0 = cl.fabric.launches, _counter(cl.client, "device_get_host_staged_total")
            ecs, got_sizes = cl.client.batch_get_device_scatter([f"o{k}" for k, *_ in items], [dst.data_ptr() + r for r in regions],
                                                                [it[1] for it in items], [it[2] for it in items], [it[3] for it in items],
                                                                _stream())
            assert ecs == [bb.ErrorCode.OK] * len(items), ecs
            assert got_sizes == [sizes[k] for k, *_ in items]
            assert _counter(cl.client, "device_get_host_staged_total") == st0 + 2  # the skewed pointer and the 33-byte gap
            assert cl.fabric.launches > l0  # the other items took the fused kernel
            torch.cuda.synchronize()
            want = np.full(dst.numel(), GUARD, dtype=np.uint8)
            for (k, w, p, _, _), r in zip(items, regions):
                want[r + rows_index(sizes[k], p, w, 0)] = objs[k]
            got = dst.cpu().numpy()
            assert np.array_equal(got, want), np.nonzero(got != want)[0][:8]
        E = bb.ErrorCode
        ecs, _ = cl.client.batch_get_device_scatter(["o3", "o3", "o3"], [dst.data_ptr()] * 3, [65, 8, 16], [64, 2**63, 48], [2, 3, 10],
                                                    _stream())
        assert ecs == [E.INVALID_ARGUMENT, E.VALUE_OUT_OF_RANGE, E.BUFFER_OVERFLOW], ecs
    finally:
        cl.stop()


def test_client_fp8_scattered_gets(bb):
    """batch_get_device_fp8_scatter against a dense fp8 get scattered by torch; a misaligned pointer and an odd gap fail
    alone with NOT_IMPLEMENTED, rows * width != n_elems with INVALID_ARGUMENT."""
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=128 << 20, cluster_id="t-scat-fp8", max_replicas=2)
    try:
        cfg = bb.WorkerConfig(replication_factor=2, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_GPU])
        shapes = [(256, 264, 64), (T, T + 8, 5), (32, 32, 100), (4096, 4096 + 16, 33)]  # (width, pitch, rows) in elements
        keys, dense = [], []
        for k, (w, p, r) in enumerate(shapes):
            t = _bf16(w * r, 70 + k)
            keys.append(f"f{k}")
            assert cl.client.batch_put_device_fp8([keys[-1]], [t.data_ptr()], [t.numel()], cfg, _stream()) == [bb.ErrorCode.OK]
            d = torch.empty_like(t)
            assert cl.client.batch_get_device_fp8([keys[-1]], [d.data_ptr()], [t.numel()], _stream()) == [bb.ErrorCode.OK]
            dense.append(d)
        outs = [torch.full((r, p), -7.0, dtype=torch.bfloat16, device="cuda") for w, p, r in shapes]
        ecs = cl.client.batch_get_device_fp8_scatter(keys, [o.data_ptr() for o in outs], [w * r for w, _, r in shapes],
                                                     [s[0] for s in shapes], [s[1] for s in shapes], [s[2] for s in shapes], _stream())
        assert ecs == [bb.ErrorCode.OK] * len(shapes), ecs
        torch.cuda.synchronize()
        for o, d, (w, p, r) in zip(outs, dense, shapes):
            assert torch.equal(o[:, :w].reshape(-1).view(torch.int16), d.view(torch.int16))
            assert bool((o[:, w:] == -7.0).all())
        E = bb.ErrorCode
        o = torch.full((64 * 300,), -7.0, dtype=torch.bfloat16, device="cuda")
        ecs = cl.client.batch_get_device_fp8_scatter(["f0"] * 4, [o.data_ptr() + 2, o.data_ptr(), o.data_ptr(), o.data_ptr()],
                                                     [256 * 64] * 4, [256, 256, 256, 256], [264, 260, 264, 264], [64, 64, 63, 64],
                                                     _stream())
        assert ecs == [E.NOT_IMPLEMENTED, E.NOT_IMPLEMENTED, E.INVALID_ARGUMENT, E.OK], ecs
    finally:
        cl.stop()


# ---------------------------------------------------------------------------------------------------- TensorStore


def test_tensor_store_get_into(bb):
    """get_into contiguous tensors and views (W[:, a:b], kv[:, :, h0:h1, :], t[::k]), a transposed view, a misaligned packed
    view and a padded packed tensor, packed and unpacked in one batch: each result equals get(key) and no element of the
    underlying storage outside the view changes."""
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id="t-scat-store")
    try:
        store = TensorStore(cl.client)
        g = torch.Generator(device="cuda").manual_seed(5)
        W = torch.randn(256, 512, device="cuda", generator=g).to(torch.bfloat16)
        kv = torch.randn(4, 2, 16, 64, device="cuda", generator=g).to(torch.bfloat16)
        ids = torch.randint(0, 1 << 30, (1000, 24), device="cuda", generator=g, dtype=torch.int32)
        # (key, tensor to store, pack_fp8, function giving the target view of a fresh base)
        cases = [("w_cols", W[:, 128:256].contiguous(), False, lambda B: B["W"][:, 128:256]),
                 ("w_cols8", W[:, 64:320].contiguous(), True, lambda B: B["W"][:, 64:320]),
                 ("kv_heads", kv[:, :, 4:12, :].contiguous(), False, lambda B: B["kv"][:, :, 4:12, :]),
                 ("kv_heads8", kv[:, :, 8:16, :].contiguous(), True, lambda B: B["kv"][:, :, 8:16, :]),
                 ("step", ids[::3].contiguous(), False, lambda B: B["ids"][::3]),
                 ("whole", W.clone(), False, lambda B: B["W"]),
                 ("whole8", W.clone(), True, lambda B: B["W"]),
                 ("T", W[:64, :32].t().contiguous(), False, lambda B: B["W"][:64, :32].t()),               # transposed: route 4
                 ("mis8", W[:, 3:35].contiguous(), True, lambda B: B["W"][:, 3:35]),                       # misaligned: route 4
                 ("pad8", torch.randn(7, 9, device="cuda", generator=g).to(torch.bfloat16), True, lambda B: B["W"][:7, :9])]
        for k, t, p, _ in cases:
            store.put(k, t, pack_fp8=p)
        refs = {k: store.get(k) for k, *_ in cases}
        bases = {"W": torch.randn(256, 512, device="cuda", generator=g).to(torch.bfloat16),
                 "kv": torch.randn(4, 2, 16, 64, device="cuda", generator=g).to(torch.bfloat16),
                 "ids": torch.randint(0, 1 << 30, (1000, 24), device="cuda", generator=g, dtype=torch.int32)}
        # one batch per group, packed and unpacked mixed; every view is of its own copy of the bases, so outs never overlap
        for group in (["w_cols", "kv_heads", "step", "whole8", "mis8"], ["w_cols8", "kv_heads8", "T", "pad8"], ["whole"]):
            sel = [c for c in cases if c[0] in group]
            Bs = [{name: t.clone() for name, t in bases.items()} for _ in sel]
            views = [fn(B) for (*_, fn), B in zip(sel, Bs)]
            outside = []  # per case: mask of every base element outside its view
            for (*_, fn), B in zip(sel, Bs):
                m = {name: torch.ones_like(t, dtype=torch.bool) for name, t in B.items()}
                fn(m).fill_(False)
                outside.append(m)
            outs = store.batch_get_into([k for k, *_ in sel], views)
            assert all(o is v for o, v in zip(outs, views))
            torch.cuda.synchronize()
            for (k, *_), v, B, m in zip(sel, views, Bs, outside):
                assert torch.equal(v, refs[k]), k
                for name in B:
                    assert torch.equal(B[name][m[name]], bases[name][m[name]]), (k, name)
        # contiguous out, alone
        out = torch.empty_like(W)
        assert store.get_into("whole", out) is out and torch.equal(out, refs["whole"])
        with pytest.raises(KeyError):
            store.get_into("missing", out)
        with pytest.raises(TypeError):
            store.get_into("whole", out.float())
        with pytest.raises(TypeError):
            store.get_into("w_cols8", torch.empty(256, 256, dtype=torch.float32, device="cuda"))
        with pytest.raises(ValueError):
            store.get_into("whole", out[:, :10])
        with pytest.raises(ValueError):
            store.get_into("whole", torch.empty(256, 512, dtype=torch.bfloat16))
    finally:
        cl.stop()


def test_get_into_async_waits_for_the_callers_stream(bb):
    from blackbird_b200.ops.tensor_store import AsyncTensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=128 << 20, cluster_id="t-scat-async")
    try:
        store = AsyncTensorStore(cl.client)
        W = torch.randn(512, 1024, device="cuda").to(torch.bfloat16)
        store.put("a", W[:, 256:768].contiguous())
        target = torch.zeros(512, 1024, dtype=torch.bfloat16, device="cuda")
        torch.cuda._sleep(100_000_000)  # the caller's stream is still busy ...
        target.fill_(3.0)                # ... and then writes the target: the get must come after this
        fut = store.get_into_async(["a"], [target[:, 256:768]])
        (out,) = fut.result(timeout=60)
        torch.cuda.synchronize()
        assert torch.equal(out, W[:, 256:768])
        assert bool((target[:, :256] == 3.0).all()) and bool((target[:, 768:] == 3.0).all())
        store.close()
    finally:
        cl.stop()
