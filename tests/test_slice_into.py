"""Slice gets into existing tensors on the GPU: the windowed scattering store (XFER_WINDOW_ROWS) of bb_xfer and of the fused
MXFP8 unpack through XferEngine, the client's batch_get_device_strided_scatter / batch_get_device_fp8_strided_scatter on a
GpuRankCluster (HBM and DRAM tiers, striped and replicated objects, fail-over), and TensorStore's slice-into methods.  A
windowed scattered descriptor stores the window's units into rows of the caller's tensor by the rule of WindowRows; the
tile in shared memory is the object's own, so every check covers the stored pieces, the guard bytes around and between
them, and the digest, which must equal that of a plain get of the same object."""
import numpy as np
import pytest
import torch
from test_mxfp8_exhaustive import model_unpack
from test_mxfp8_wide import model_unpack_w

pytestmark = pytest.mark.gpu

T = 16384
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


def _random(bb, n, seed):
    t = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
    bb.random_fill(t.data_ptr(), t.numel(), seed, _stream())
    return t


def model_pairs(offset, width, pitch, rows, dw, dp, dph=0):
    """(object index, destination index) of every stored unit (the independent model of tests/test_slice_into_cpu.py)."""
    r = np.arange(rows, dtype=np.int64)[:, None]
    c = np.arange(width, dtype=np.int64)[None, :]
    x = (offset + r * pitch + c).ravel()
    q = (r * width + c).ravel() + dph
    return x, (q // dw) * dp + q % dw


# (object bytes, (offset, width, pitch, rows), (dst width, dst pitch, dst phase)): ranges and strided windows, tail tiles,
# destination rows narrower and wider than the window's, heads and tails under 16 bytes, thousands of short pieces a tile
SPECS = [(3 * T + 5, (100, 2 * T, 2 * T, 1), (1000, 1048, 0)),
         (4 * T, (64, 4096, 8192, 8), (4096, 4096 + 512, 0)),
         (4 * T, (16, 1024, 4096, 16), (512, 2048, 0)),
         (2 * T + 100, (3, 5, 21, 1500), (7, 23, 0)),
         (2 * T, (0, 48, 64, 500), (4096 + 3, 8192 + 3, 0)),
         (T, (5, 777, 777, 1), (100, 116, 37)),
         (8 * T, (0, 8 * T, 8 * T, 1), (T + 8, T + 8 + 48, 8))]


def _place(specs):
    """Destination regions in one buffer: each region's base congruent so that its first stored byte is co-aligned."""
    regions, o = [], 64
    for n, (off, w, p, r), (dw, dp, dph) in specs:
        x0, d0 = model_pairs(off, w, p, r, dw, dp, _phase(off, w, p, r, dph))
        o += (int(x0[0]) - int(d0[0]) - o) % 16
        regions.append(o)
        o += int(d0.max()) + 1 + 64
    return regions, o + 64


def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


def _window(off, w, p, r):
    return (off, off + (r - 1) * p + w) if r == 1 or w == p else (off, off + (r - 1) * p + w, p, w, (p - off % p) % p)


def _phase(off, w, p, r, dph=0):
    """The destination phase the engine items' windows give: a strided window without `row` counts the result from
    pattern row 0, ceil(off / p) rows before the first row read, so the result starts that many rows of w in."""
    return dph if r == 1 or w == p else dph + (off + (p - off % p) % p) // p * w


@pytest.mark.parametrize("algo", ALGOS)
def test_windowed_scatters_at_every_grid_mixed_with_other_items(bb, eng, algo):
    A = getattr(bb.ChecksumAlgo, algo)
    srcs = [_random(bb, n, 10 + k) for k, (n, *_) in enumerate(SPECS)]
    host = [s.cpu().numpy()[:n] for s, (n, *_) in zip(srcs, SPECS)]
    regions, total = _place(SPECS)
    plain_out = [torch.empty(n, dtype=torch.uint8, device="cuda") for n, *_ in SPECS]
    pdg, pst, _ = eng.run([(s.data_ptr(), o.data_ptr(), n) for s, o, (n, *_) in zip(srcs, plain_out, SPECS)], A, _stream())
    dst = torch.full((total,), GUARD, dtype=torch.uint8, device="cuda")
    extra = torch.full((3 * T + 64,), GUARD, dtype=torch.uint8, device="cuda")
    flags = bb.XFER_VERIFY if algo != "NONE" else 0
    items = []
    for s, reg, dg, (n, (off, w, p, r), (dw, dp, dph)) in zip(srcs, regions, pdg, SPECS):
        items.append((s.data_ptr(), dst.data_ptr() + reg, n, dg, flags, 0, _window(off, w, p, r), None, None, None, None, None, None,
                      (dp, dw, dph)))
    # the existing item kinds in the same batch: a plain get, a range get and a scattered get
    items += [(srcs[0].data_ptr(), extra.data_ptr(), 3 * T + 5, pdg[0], flags),
              (srcs[1].data_ptr(), extra.data_ptr() - 16, 1000, 0, 0, 0, (16, 1000)),
              (srcs[2].data_ptr(), extra.data_ptr() + 2 * T, 1000, 0, 0, 0, None, None, (128, 96, 0))]
    for g in GRIDS:
        eng.set_max_ctas(_grid(g))
        dst.fill_(GUARD)
        dg, st, _ = eng.run(items, A, _stream())
        assert dg[: len(SPECS)] == list(pdg), g
        assert st[: len(SPECS)] == [0] * len(SPECS), g
        torch.cuda.synchronize()
        want = np.full(total, GUARD, dtype=np.uint8)
        for reg, h, (n, (off, w, p, r), (dw, dp, dph)) in zip(regions, host, SPECS):
            x, d = model_pairs(off, w, p, r, dw, dp, _phase(off, w, p, r, dph))
            want[reg + d] = h[x]
        got = dst.cpu().numpy()
        assert np.array_equal(got, want), (algo, g, np.nonzero(got != want)[0][:8])
    if algo != "NONE":  # a wrong digest is a mismatch and the engine still stores nothing outside the rows
        bad = [it[:3] + (it[3] ^ 1,) + it[4:] for it in items[: len(SPECS)]]
        _, st, _ = eng.run(bad, A, _stream())
        assert st == [1] * len(SPECS)


def test_inline_and_single_item_batches(bb, eng):
    src = _random(bb, 2 * T, 3)
    h = src.cpu().numpy()[: 2 * T]
    dst = torch.full((4 * T,), GUARD, dtype=torch.uint8, device="cuda")
    for r, (off, w, p, rows), (dw, dp) in [(1, (32, 96, 160, 100), (64, 96)), (1, (0, 100, 100, 1), (16, 48))]:
        eng.run([(src.data_ptr(), dst.data_ptr() + 64, 2 * T, 0, 0, 0, _window(off, w, p, rows), None, None, None, None, None, None,
                  (dp, dw, 0))], bb.ChecksumAlgo.XXH3, _stream())
        torch.cuda.synchronize()
        want = np.full(4 * T, GUARD, dtype=np.uint8)
        x, d = model_pairs(off, w, p, rows, dw, dp, _phase(off, w, p, rows))
        want[64 + d] = h[x]
        assert np.array_equal(dst.cpu().numpy(), want)
        dst.fill_(GUARD)


def test_refusals_before_launch(bb, eng):
    src = _random(bb, 4 * T, 1)
    dst = torch.full((4 * T,), GUARD, dtype=torch.uint8, device="cuda")
    s, d = src.data_ptr(), dst.data_ptr()
    A = bb.ChecksumAlgo.XXH3
    la = eng.launches
    bad = [((s, d, 1000, 0, bb.XFER_WINDOW_ROWS, 0, (0, 500)), "INVALID_ARGUMENT"),                      # the engine's flag
           ((s, d, 1000, 0, bb.XFER_WINDOW_ROWS), "INVALID_ARGUMENT"),
           ((s, d, 1000, 0, 0, 0, (0, 500), None, None, None, None, None, None, (100, 0, 0)), "INVALID_ARGUMENT"),   # width 0
           ((s, d, 1000, 0, 0, 0, (0, 500), None, None, None, None, None, None, (100, 101, 0)), "INVALID_ARGUMENT"),
           ((s, d, 1000, 0, 0, 0, (0, 500), None, None, None, None, None, None, (100, 50, 50)), "INVALID_ARGUMENT"),
           ((s, [d, d + T], 1000, 0, 0, 0, (0, 500), None, None, None, None, None, None, (128, 96, 0)), "INVALID_ARGUMENT"),
           ((s, d, 1000, 0, 0, 0, (0, 500), None, (128, 96, 0), None, None, None, None, (128, 96, 0)), "INVALID_ARGUMENT"),
           ((s, d + 4, 1000, 0, 0, 0, (0, 500), None, None, None, None, None, None, (128, 96, 0)), "INVALID_ADDRESS"),
           ((s, d, 1000, 0, 0, 0, (0, 500), None, None, None, None, None, None, (120, 96, 0)), "INVALID_ADDRESS"),  # gap 24
           ((s, d, 4000, 0, 0, 0, (0, 4000, 100, 64, 0), None, None, None, None, None, None, (128, 96, 0)), "INVALID_ADDRESS")]
    for it, err in bad:
        with pytest.raises(RuntimeError, match=err):
            eng.run([it], A, _stream())
    assert eng.launches == la
    torch.cuda.synchronize()
    assert bool((dst == GUARD).all())


def _wide(n, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(n, device="cuda", generator=g) * 3).to(dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_fused_unpack_window_rows_bit_exact(bb, eng, dtype):
    wide = {torch.bfloat16: bb.MxWide.BF16, torch.float16: bb.MxWide.F16, torch.float32: bb.MxWide.F32}[dtype]
    es = torch.tensor([], dtype=dtype).element_size()
    g = 16 // es
    # (n_elems, (offset, width, pitch, rows), (dst width, dst pitch)) in elements; the last two windows hold the whole
    # object (one range, and rows that touch), which the engine takes as the object's own rows, in the same launch
    specs = [(4 * T, (8 * g, 256, 1024, 40), (256, 256 + 4 * g)), (2 * T + 64, (0, 5000, 5000, 1), (1000, 1000 + g)),
             (T, (g, 64, 128, 100), (32, 32 + 2 * g)), (8 * T, (0, 4 * T, 8 * T, 1), (T + g, T + 3 * g)),
             (2 * T, (0, 2 * T, 2 * T, 1), (512, 512 + 2 * g)), (T, (0, 256, 256, T // 256), (1024, 1024 + g))]
    packed, refs = [], []
    for k, (n, *_) in enumerate(specs):
        w = _wide(n, dtype, k)
        p = torch.empty(n + n // 32, dtype=torch.uint8, device="cuda")
        bb.mxfp8_pack(w.data_ptr(), n, p.data_ptr(), _stream(), wide=wide)
        packed.append(p)
        # the reference values: the exact host model of the format (tests/test_mxfp8_exhaustive.py, test_mxfp8_wide.py)
        host = p.cpu().numpy()
        bits = model_unpack(host, n) if dtype == torch.bfloat16 else model_unpack_w(host, n, "f16" if dtype == torch.float16 else "f32")
        refs.append(np.ascontiguousarray(bits).view(np.uint8).reshape(n, es))
    plain = [torch.empty(n, dtype=dtype, device="cuda") for n, *_ in specs]
    pdg, pst, _ = eng.run_fp8([(t.data_ptr(), p.data_ptr(), n) for t, p, (n, *_) in zip(plain, packed, specs)], True, _stream(), wide=wide)
    regions, o = [], 64
    for n, (off, w, p, r), (dw, dp) in specs:
        x0, d0 = model_pairs(off, w, p, r, dw, dp, _phase(off, w, p, r))
        o += (int(x0[0]) - int(d0[0]) - o) % g  # the first stored element's destination co-aligned
        regions.append(o)
        o += int(d0.max()) + 1 + 64
    dst = torch.full((o * es + 64,), GUARD, dtype=torch.uint8, device="cuda")
    items = [(dst.data_ptr() + es * reg, p.data_ptr(), n, dg, _window(off, w, pi, r), None, None, None, None, None, None, None, (dp, dw, 0))
             for reg, p, dg, (n, (off, w, pi, r), (dw, dp)) in zip(regions, packed, pdg, specs)]
    for gr in (1, "sms"):
        eng.set_max_ctas(_grid(gr))
        dst.fill_(GUARD)
        dg, st, _ = eng.run_fp8(items, True, _stream(), wide=wide)
        assert st == [0] * len(specs) and dg == pdg
        torch.cuda.synchronize()
        want = np.full((o * es + 64,), GUARD, dtype=np.uint8)
        for reg, ref, (n, (off, w, p, r), (dw, dp)) in zip(regions, refs, specs):
            x, d = model_pairs(off, w, p, r, dw, dp, _phase(off, w, p, r))
            want[((reg + d)[:, None] * es + np.arange(es)).ravel()] = ref[x].ravel()
        assert np.array_equal(dst.cpu().numpy(), want), gr
    with pytest.raises(RuntimeError, match="INVALID_ADDRESS"):
        eng.run_fp8([(items[0][0] + 2,) + items[0][1:]], True, _stream(), wide=wide)


def test_client_slice_gets_hbm_dram_striped_and_failover(bb):
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=128 << 20, cluster_id="t-slice-into", dram_bytes=64 << 20, max_replicas=3)
    try:
        A = bb.ChecksumAlgo.XXH3
        striped = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=2, ttl_ms=0, min_shard_size=4096, checksum=A,
                                  preferred_classes=[bb.StorageClass.RAM_GPU, bb.StorageClass.RAM_CPU])
        plain = bb.WorkerConfig(replication_factor=2, max_workers_per_copy=1, ttl_ms=0, checksum=A, preferred_classes=[bb.StorageClass.RAM_GPU])
        dram = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, checksum=A, preferred_classes=[bb.StorageClass.RAM_CPU])
        sizes, cfgs, objs = [1 << 20, 1 << 20, 1 << 20], [striped, plain, dram], []
        for k, (n, cfg) in enumerate(zip(sizes, cfgs)):
            t = _random(bb, n, 70 + k)
            assert cl.client.batch_put_device([f"o{k}"], [t.data_ptr()], [n], cfg, _stream()) == [bb.ErrorCode.OK]
            objs.append(t.cpu().numpy()[:n])
        # (key, offset, width, pitch, rows, dst width, dst pitch, skew)
        items = [(0, 64, 4096, 8192, 100, 4096, 4096 + 1024, 0), (1, 0, 1 << 19, 1 << 19, 1, 1000, 1040, 0),
                 (2, 16, 1024, 4096, 200, 512, 2048, 0), (1, 3, 5, 21, 2000, 7, 23, 1), (0, 0, 1 << 20, 1 << 20, 1, 65536, 65536 + 48, 0)]
        regions, o = [], 64
        for k, off, w, p, r, dw, dp, sk in items:
            x, d = model_pairs(off, w, p, r, dw, dp)
            o += (int(x[0]) - int(d[0]) - o) % 16 + sk
            regions.append(o)
            o += int(d.max()) + 64
        dst = torch.full((o + 64,), GUARD, dtype=torch.uint8, device="cuda")
        for rep in range(2):
            if rep == 1:  # corrupt copy 0 of o1 (every copy is local: it is read first) in a gap: the get fails over
                sh = cl.client.get_workers("o1")[0].shards[0]
                be = cl.worker.backend(sh.pool_id)
                be.write(sh.offset + 900000, bytes([be.read(sh.offset + 900000, 1)[0] ^ 0xFF]))
                fo = _counter(cl.client, "replica_failover_total")
            dst.fill_(GUARD)
            ecs = cl.client.batch_get_device_strided_scatter([f"o{it[0]}" for it in items], [dst.data_ptr() + r for r in regions],
                                                             *[[it[j] for it in items] for j in range(1, 7)], _stream())
            assert ecs == [bb.ErrorCode.OK] * len(items), ecs
            torch.cuda.synchronize()
            want = np.full(o + 64, GUARD, dtype=np.uint8)
            for reg, (k, off, w, p, r, dw, dp, sk) in zip(regions, items):
                x, d = model_pairs(off, w, p, r, dw, dp)
                want[reg + d] = objs[k][x]
            got = dst.cpu().numpy()
            assert np.array_equal(got, want), np.nonzero(got != want)[0][:8]
        assert _counter(cl.client, "replica_failover_total") > fo
        assert _counter(cl.client, "device_get_host_staged_total") >= 1  # the odd-gap item
    finally:
        cl.stop()


def test_tensor_store_slice_into(bb):
    """Every slice-into method with canaries around each view: only the view's elements change, and each equals the
    stored tensor's slice; a TP column shard lands in its columns of a fused parameter."""
    from blackbird_b200.ops.tensor_store import AsyncTensorStore, TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id="t-slice-store")
    try:
        store = TensorStore(cl.client)
        g = torch.Generator(device="cuda").manual_seed(9)
        W = torch.randn(512, 1024, device="cuda", generator=g).to(torch.bfloat16)
        kv = torch.randn(8, 16, 128, device="cuda", generator=g).to(torch.float16)
        v = torch.randn(4096, device="cuda", generator=g)
        store.batch_put(["W", "kv", "v"], [W, kv, v])
        store.batch_put(["Wp", "kvp"], [W, kv], pack_fp8=True)
        Wq = store.get("Wp")
        kvq = store.get("kvp")
        # a fused QKV parameter: the stored W's columns [256, 512) land in columns [1024, 1280) of a 3x wider parameter
        for key, ref in (("W", W), ("Wp", Wq)):
            fused = torch.full((512, 3 * 1024), 7.0, device="cuda", dtype=torch.bfloat16)
            before = fused.clone()
            out = fused[:, 1024:1280]
            store.get_slice_into(key, out, 1, 256, 512)
            assert torch.equal(out, ref[:, 256:512])
            before[:, 1024:1280] = ref[:, 256:512]
            assert torch.equal(fused, before)
        # heads h0:h1 of a stored layer into the same heads of a live buffer; dim 0 rows; a contiguous out; a transposed out
        for key, ref in (("kv", kv), ("kvp", kvq)):
            live = torch.full((8, 16, 128), -1.0, device="cuda", dtype=torch.float16)
            before = live.clone()
            store.get_slice_into(key, live[:, 4:12, :], 1, 4, 12)
            before[:, 4:12] = ref[:, 4:12]
            assert torch.equal(live, before)
        buf = torch.full((5000,), 3.0, device="cuda")
        store.get_rows_into("v", buf[100:1124], 1000, 2024)
        want = torch.full((5000,), 3.0, device="cuda")
        want[100:1124] = v[1000:2024]
        assert torch.equal(buf, want)
        outs = [torch.empty(512, 64, device="cuda", dtype=torch.bfloat16), torch.full((64, 512), 2.0, device="cuda", dtype=torch.bfloat16).t(),
                torch.full((512, 200), 1.0, device="cuda", dtype=torch.bfloat16)[:, 3:67]]
        store.batch_get_slices_into(["W", "W", "Wp"], outs, [1, -1, 1], [0, 64, 128], [64, 128, 192])
        assert torch.equal(outs[0], W[:, :64]) and torch.equal(outs[1], W[:, 64:128]) and torch.equal(outs[2], Wq[:, 128:192])
        rows = torch.zeros(300, 1024, device="cuda", dtype=torch.bfloat16)
        store.batch_get_rows_into(["W"], [rows[10:110]], [200], [300])
        assert torch.equal(rows[10:110], W[200:300]) and not rows[:10].any() and not rows[110:].any()
        # packed windows that hold the whole object, into row views, in one call with a partial one: all three take the
        # fused call (no fallback), and only the views change
        n0 = _counter(cl.client, "device_get_fp8_strided_scatter_total")
        fused = torch.full((512, 3 * 1024), 7.0, device="cuda", dtype=torch.bfloat16)
        part = torch.full((512, 256), 5.0, device="cuda", dtype=torch.bfloat16)
        big = torch.full((8, 16, 256), -3.0, device="cuda", dtype=torch.float16)
        store.batch_get_slices_into(["Wp", "Wp", "kvp"], [fused[:, 1024:2048], part[:, 64:128], big[:, :, :128]], [1, 1, 0], [0, 128, 0],
                                    [1024, 192, 8])
        assert _counter(cl.client, "device_get_fp8_strided_scatter_total") == n0 + 3
        want = torch.full_like(fused, 7.0)
        want[:, 1024:2048] = Wq
        assert torch.equal(fused, want)
        want = torch.full_like(part, 5.0)
        want[:, 64:128] = Wq[:, 128:192]
        assert torch.equal(part, want)
        want = torch.full_like(big, -3.0)
        want[:, :, :128] = kvq
        assert torch.equal(big, want)
        a = AsyncTensorStore(cl.client)
        try:
            tgt = torch.zeros(512, 2048, device="cuda", dtype=torch.bfloat16)
            a.get_slices_into_async(["W"], [tgt[:, 512:768]], [1], [0], [256]).result()
            assert torch.equal(tgt[:, 512:768], W[:, :256]) and not tgt[:, :512].any() and not tgt[:, 768:].any()
        finally:
            a.close()
        with pytest.raises(ValueError):
            store.get_slice_into("W", torch.empty(512, 10, device="cuda", dtype=torch.bfloat16), 1, 0, 11)
    finally:
        cl.stop()
