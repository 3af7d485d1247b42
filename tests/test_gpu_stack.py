"""GPU tests: fused kernels against CPU models and the full client -> keystone -> GPU worker path."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need CUDA (marked gpu)")
    return torch


def _stream(torch):
    return torch.cuda.current_stream().cuda_stream


@pytest.mark.parametrize("algo_name", ["BBH64", "CRC32C", "XXH3"])
@pytest.mark.parametrize("n", [16, 255 * 16, 16384, 16385, 100000, (1 << 20) + 7, 5 << 20])
def test_fused_digest_matches_cpu_model(bb, torch_cuda, algo_name, n):
    torch = torch_cuda
    algo = getattr(bb.ChecksumAlgo, algo_name)
    eng = bb.XferEngine(0, 1024, 2)
    src = torch.randint(0, 256, (n + 64,), dtype=torch.uint8, device="cuda")[:n]
    dst = torch.full((n + 64,), 0xAB, dtype=torch.uint8, device="cuda")
    dg, st, ms = eng.run([(src.data_ptr(), dst.data_ptr(), n)], algo, _stream(torch))
    torch.cuda.synchronize()
    host = src.cpu().numpy()
    ref = bb.bbh64(host) if algo_name == "BBH64" else bb.xxh3t64(host) if algo_name == "XXH3" else bb.crc32c(host)
    assert dg[0] == ref
    assert torch.equal(src, dst[:n]) and bool((dst[n:] == 0xAB).all())


def test_fused_verify_and_fanout(bb, torch_cuda):
    torch = torch_cuda
    eng = bb.XferEngine(0, 1024, 2)
    n = 3 * bb.TILE_BYTES + 4096
    src = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda")
    dsts = [torch.zeros(n, dtype=torch.uint8, device="cuda") for _ in range(3)]
    ref = bb.bbh64(src.cpu().numpy())
    dg, st, _ = eng.run([(src.data_ptr(), [d.data_ptr() for d in dsts], n, ref, bb.XFER_VERIFY)], bb.ChecksumAlgo.BBH64, _stream(torch))
    assert dg[0] == ref and st[0] == 0
    assert all(torch.equal(src, d) for d in dsts)
    dg, st, _ = eng.run([(src.data_ptr(), dsts[0].data_ptr(), n, ref ^ 0x10, bb.XFER_VERIFY)], bb.ChecksumAlgo.BBH64, _stream(torch))
    assert st[0] == 1  # CHECKSUM_MISMATCH detected on device


def test_fused_batch_of_small_objects(bb, torch_cuda):
    torch = torch_cuda
    eng = bb.XferEngine(0, 8192, 2)
    nobj, osz = 2048, 1024
    big = torch.randint(0, 256, (nobj * osz,), dtype=torch.uint8, device="cuda")
    out = torch.zeros_like(big)
    items = [(big.data_ptr() + i * osz, out.data_ptr() + i * osz, osz) for i in range(nobj)]
    dg, st, _ = eng.run(items, bb.ChecksumAlgo.BBH64, _stream(torch))
    h = big.cpu().numpy()
    assert all(dg[i] == bb.bbh64(h[i * osz:(i + 1) * osz]) for i in range(0, nobj, 97))
    assert torch.equal(big, out)


@pytest.mark.parametrize("algo_name", ["BBH64", "CRC32C", "XXH3", "NONE"])
def test_small_object_warp_path_matches_cpu_models_and_the_big_kernel(bb, torch_cuda, algo_name):
    """xfer_small.cu: batches made only of objects <= 4 KiB take the warp-per-object kernel; bytes and digests are
    identical to the CPU models and to what the TMA / wgmma kernel produces for the same objects."""
    torch = torch_cuda
    algo = getattr(bb.ChecksumAlgo, algo_name)
    eng = bb.XferEngine(0, 8192, 2)
    sizes = [1, 3, 15, 16, 17, 31, 64, 100, 127, 128, 129, 255, 256, 1000, 1024, 2047, 2048, 3000, 4080, 4095, 4096] + [((7 * i) % 4096) + 1 for i in range(300)]
    stride = 4096 + 256
    n = len(sizes)
    src = torch.randint(0, 256, (n * stride,), dtype=torch.uint8, device="cuda")
    outs = [torch.full((n * stride,), 0xCD, dtype=torch.uint8, device="cuda") for _ in range(2)]
    items = [(src.data_ptr() + i * stride, [o.data_ptr() + i * stride for o in outs], sz) for i, sz in enumerate(sizes)]
    before = eng.small_launches
    dg, st, _ = eng.run(items, algo, _stream(torch))
    assert eng.small_launches == before + 1  # the warp path really ran
    torch.cuda.synchronize()
    h = src.cpu().numpy()
    for i, sz in enumerate(sizes):
        blob = h[i * stride:i * stride + sz]
        if algo_name != "NONE":
            assert dg[i] == (bb.bbh64(blob) if algo_name == "BBH64" else bb.xxh3t64(blob) if algo_name == "XXH3" else bb.crc32c(blob)), (i, sz)
        for o in outs:
            assert torch.equal(o[i * stride:i * stride + sz], src[i * stride:i * stride + sz]), (i, sz)
            assert bool((o[i * stride + sz:(i + 1) * stride] == 0xCD).all()), (i, sz)  # nothing written past the object
    if algo_name == "NONE":
        return
    # same objects through the big kernel: identical digests (the keystone cannot tell the paths apart)
    eng.set_small_path(False)
    dg2, _, _ = eng.run(items, algo, _stream(torch))
    assert eng.small_launches == before + 1 and list(dg2) == list(dg)
    eng.set_small_path(True)
    # verify on get: a flipped bit in the stored copy is reported per object
    outs[0][5 * stride + 2] ^= 1
    back = torch.zeros_like(src)
    gets = [(outs[0].data_ptr() + i * stride, back.data_ptr() + i * stride, sz, dg[i], bb.XFER_VERIFY) for i, sz in enumerate(sizes)]
    _, st, _ = eng.run(gets, algo, _stream(torch))
    assert st[5] == 1 and sum(st) == 1
    # single object: descriptors travel in the kernel parameters, results land in pinned memory
    dg1, st1, ms = eng.run([items[20]], algo, _stream(torch))
    assert dg1[0] == dg[20] and st1[0] == 0


def test_mailbox_resident_warp_serves_single_small_objects_without_a_launch(bb, torch_cuda):
    """xfer_small.cu bb_mailbox_kernel: a lingering resident warp fed through pinned memory.  Same bytes and digests as the
    launched paths; stays resident across back-to-back requests (no launch), sees fresh source data every time (volatile
    loads: L1 is not invalidated inside a resident kernel), leaves by itself after the linger time and comes back on the
    next request; device-wide synchronisation never waits for more than the linger time."""
    import time

    torch = torch_cuda
    eng = bb.XferEngine(0, 256, 2)
    s = _stream(torch)
    src = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    dst = torch.zeros(4096 + 64, dtype=torch.uint8, device="cuda")
    algos = [("XXH3", bb.xxh3t64), ("BBH64", bb.bbh64), ("CRC32C", bb.crc32c), ("NONE", None)]
    l0, r0 = eng.mailbox_launches, eng.mailbox_requests
    n_req = 0
    for rnd in range(40):
        name, ref = algos[rnd % 4]
        n = [1, 17, 256, 1000, 4095, 4096][rnd % 6]
        src.copy_(torch.randint(0, 256, (4096,), dtype=torch.uint8, device="cuda"))  # same address, new contents every round
        dst.fill_(0xEE)
        torch.cuda.current_stream().synchronize()  # the mailbox is only used when the stream has nothing pending
        dg, st, _ = eng.run([(src.data_ptr(), dst.data_ptr(), n)], getattr(bb.ChecksumAlgo, name), s)
        n_req += 1
        host = src[:n].cpu().numpy()
        if ref is not None:
            assert dg[0] == ref(host), (rnd, name, n)
        assert torch.equal(dst[:n], src[:n]) and bool((dst[n:] == 0xEE).all()), (rnd, name, n)
    assert eng.mailbox_requests == r0 + n_req
    # (each round spends a few hundred microseconds in torch between requests, so the warp lingers out now and then;
    # back-to-back requests below must all be served by one incarnation)
    assert eng.mailbox_launches - l0 < n_req
    l_b2b = eng.mailbox_launches
    for _ in range(50):
        eng.run([(src.data_ptr(), dst.data_ptr(), 4096)], bb.ChecksumAlgo.XXH3, s)
    assert eng.mailbox_launches - l_b2b <= 1, "the warp should have stayed resident across back-to-back requests"
    n_req += 50
    # verify flag travels through the mailbox too
    good = bb.xxh3t64(src.cpu().numpy())
    _, st, _ = eng.run([(src.data_ptr(), dst.data_ptr(), 4096, good ^ 1, bb.XFER_VERIFY)], bb.ChecksumAlgo.XXH3, s)
    assert st[0] == 1
    # a batch of 8 small objects is 8 mailbox requests; 9 go through the launched warp-per-object kernel
    many = torch.randint(0, 256, (9 * 4096,), dtype=torch.uint8, device="cuda")
    out = torch.zeros_like(many)
    torch.cuda.synchronize()
    r1, sl1 = eng.mailbox_requests, eng.small_launches
    dg8, _, _ = eng.run([(many.data_ptr() + i * 4096, out.data_ptr() + i * 4096, 3000 + i) for i in range(8)], bb.ChecksumAlgo.CRC32C, s)
    assert eng.mailbox_requests == r1 + 8 and eng.small_launches == sl1
    dg9, _, _ = eng.run([(many.data_ptr() + i * 4096, out.data_ptr() + i * 4096, 3000 + i) for i in range(9)], bb.ChecksumAlgo.CRC32C, s)
    assert eng.mailbox_requests == r1 + 8 and eng.small_launches == sl1 + 1 and list(dg9[:8]) == list(dg8)
    h = many.cpu().numpy()
    assert all(dg9[i] == bb.crc32c(h[i * 4096:i * 4096 + 3000 + i]) for i in range(9))
    # work pending on the stream -> not the mailbox (ordering with the caller's stream would be lost)
    big = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    r2 = eng.mailbox_requests
    big.fill_(7)
    big.fill_(8)
    eng.run([(src.data_ptr(), dst.data_ptr(), 4096)], bb.ChecksumAlgo.XXH3, s)
    torch.cuda.synchronize()
    # (either path is correct; when the fills were still running the request must have been launched)
    assert eng.mailbox_requests - r2 in (0, 1)
    # linger: the warp leaves on its own; a device-wide sync is quick; the next request brings it back
    t0 = time.perf_counter()
    torch.cuda.synchronize()
    assert time.perf_counter() - t0 < 0.05
    time.sleep(0.3)
    l1 = eng.mailbox_launches
    dg, _, _ = eng.run([(src.data_ptr(), dst.data_ptr(), 4096)], bb.ChecksumAlgo.XXH3, s)
    assert dg[0] == good and eng.mailbox_launches == l1 + 1
    # engines can be dropped while their warp still lingers
    del eng


def test_standalone_crc32c_kernel(bb, torch_cuda):
    torch = torch_cuda
    for n in [1, 511, 513, 100001]:
        src = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda")
        out = torch.zeros(1, dtype=torch.int32, device="cuda")
        scratch = torch.zeros(n // 512 + 2, dtype=torch.int32, device="cuda")
        bb.crc32c_device(src.data_ptr(), n, out.data_ptr(), scratch.data_ptr(), _stream(torch))
        torch.cuda.synchronize()
        assert (int(out.item()) & 0xFFFFFFFF) == bb.crc32c(src.cpu().numpy())


def test_full_stack_put_get_gpu_tier(bb, torch_cuda):
    """client SDK -> keystone (placement, PENDING->COMPLETE, digests) -> GPU slab via fused kernels."""
    torch = torch_cuda
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=512 << 20, cluster_id="t-gpu")
    try:
        n, size = 16, (1 << 20) + 48
        stride = ((size + 255) // 256) * 256
        src = torch.randint(0, 256, (n * stride,), dtype=torch.uint8, device="cuda")
        out = torch.zeros_like(src)
        keys = [f"k{i}" for i in range(n)]
        cfg = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, preferred_classes=[bb.StorageClass.RAM_GPU])
        s = _stream(torch)
        ecs = cl.client.batch_put_device(keys, [src.data_ptr() + i * stride for i in range(n)], [size] * n, cfg, s)
        assert all(e == bb.ErrorCode.OK for e in ecs)
        ecs, sizes = cl.client.batch_get_device(keys, [out.data_ptr() + i * stride for i in range(n)], [stride] * n, s)
        assert all(e == bb.ErrorCode.OK for e in ecs) and sizes == [size] * n
        torch.cuda.synchronize()
        for i in range(n):
            assert torch.equal(src[i * stride:i * stride + size], out[i * stride:i * stride + size])
        copies = cl.client.get_workers(keys[3])
        sh = copies[0].shards[0]
        assert sh.storage_class == bb.StorageClass.RAM_GPU and sh.location["kind"] == "gpu"
        assert sh.checksum == bb.bbh64(src[3 * stride:3 * stride + size].cpu().numpy())
        # the same object is reachable through the slow path (TCP data server -> cudaMemcpy D2H)
        host_client = bb.BlackbirdClient(cl.client_api, bb.BlackbirdClientOptions(node_id="host"))
        assert host_client.get(keys[3]) == bytes(src[3 * stride:3 * stride + size].cpu().numpy())
        # corruption in the slab is detected by the fused get (digest mismatch -> CHECKSUM_MISMATCH)
        be = cl.worker.backend("hbm0")
        be.write(sh.offset + 100, b"\xff\x00\xff\x00")
        ecs, _ = cl.client.batch_get_device([keys[3]], [out.data_ptr()], [stride], s)
        assert ecs[0] == bb.ErrorCode.CHECKSUM_MISMATCH
        assert cl.client.batch_remove(keys) == [bb.ErrorCode.OK] * n
        assert cl.fabric.launches >= 3
        # per-path payload counters (Prometheus): everything here stayed in this GPU's own HBM
        assert cl.fabric.path_bytes(True, 0) == n * size and cl.fabric.path_bytes(False, 0) >= n * size
        assert cl.fabric.path_bytes(True, 1) == 0 and cl.fabric.path_bytes(True, 2) == 0
        assert 'bb_fabric_bytes_total{gpu="0",dir="put",path="hbm"} %d' % (n * size) in cl.client.metrics_text()
    finally:
        cl.stop()


def test_tensor_store_roundtrip_and_mxfp8(bb, torch_cuda):
    torch = torch_cuda
    from blackbird_b200.ops import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id="t-ts")
    try:
        ts = TensorStore(cl.client)
        a = torch.randn(257, 129, device="cuda", dtype=torch.float32)
        b = torch.randint(-5, 5, (1000,), device="cuda", dtype=torch.int32)
        ts.batch_put(["a", "b"], [a, b])
        ga, gb = ts.batch_get(["a", "b"])
        assert ga.dtype == a.dtype and ga.shape == a.shape and torch.equal(ga, a) and torch.equal(gb, b)
        kv = (torch.randn(4, 1000, 33, device="cuda") * 3).to(torch.bfloat16)  # numel not a multiple of 32
        ts.put("kv", kv, pack_fp8=True)
        sh = cl.client.get_workers("kv")[0].shards[0]
        assert sh.length == bb.mxfp8_packed_bytes((kv.numel() + 31) // 32 * 32)  # ~0.52x of the bf16 bytes in the slab
        back = ts.get("kv")
        assert back.shape == kv.shape and back.dtype == torch.bfloat16
        err = (back.float() - kv.float()).abs().max().item()
        assert err <= kv.float().abs().max().item() * 2 ** -3
        ts.remove(["a", "b", "kv"])
        assert cl.client.object_exists("kv") is False
    finally:
        cl.stop()


def test_large_batch_is_pipelined_in_chunks(bb, torch_cuda):
    """Batches >= 512 MiB are split so chunk k's kernel overlaps the Keystone round trips of chunk k+1."""
    torch = torch_cuda
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=3 << 30, cluster_id="t-chunk")
    try:
        n, size = 16, 64 << 20
        src = torch.empty(n * size, dtype=torch.uint8, device="cuda")
        bb.random_fill(src.data_ptr(), n * size, 5, 0)
        out = torch.zeros_like(src)
        keys = [f"c{i}" for i in range(n)]
        cfg = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, preferred_classes=[bb.StorageClass.RAM_GPU])
        s = _stream(torch)
        cl.client.set_device_pipeline_chunks(4)  # default: adaptive, an in-process keystone is too fast to be worth a split
        l0 = cl.fabric.launches
        assert cl.client.batch_put_device(keys, [src.data_ptr() + i * size for i in range(n)], [size] * n, cfg, s) == [bb.ErrorCode.OK] * n
        assert cl.fabric.launches - l0 == 4  # 1 GiB in four 256 MiB chunks
        ecs, sizes = cl.client.batch_get_device(keys, [out.data_ptr() + i * size for i in range(n)], [size] * n, s)
        assert ecs == [bb.ErrorCode.OK] * n and cl.fabric.launches - l0 == 8
        torch.cuda.synchronize()
        assert torch.equal(src, out)
        assert cl.client.get_workers(keys[5])[0].shards[0].checksum == bb.bbh64(src[5 * size:6 * size].cpu().numpy())
    finally:
        cl.stop()


def test_gpu_tier_spill_gpu_to_dram_to_nvme(bb, torch_cuda, tmp_path):
    """BASELINE config #4 on the GPU tier: HBM over the watermark -> LRU objects demoted to DRAM, DRAM over the
    watermark -> demoted to NVMe; soft-pinned objects stay in HBM; the device API reads demoted objects back
    bit-exact (host-staged path), and the digests recorded at put time survive both moves."""
    torch = torch_cuda
    from blackbird_b200.models.workloads import tier_spill
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id="t-spill", dram_bytes=64 << 20, nvme_bytes=256 << 20,
                        nvme_path=str(tmp_path), high_watermark=0.5, eviction_ratio=0.5)
    try:
        r = tier_spill(cl, nobj=10, size=6 << 20)
        assert r["demoted_to_dram"] >= 3 and r["demoted_to_nvme"] >= 1, r
        assert r["pinned_tier"] == "RAM_GPU" and r["verified"] == 11 and r["gpu_util_after"] <= 0.55, r
        # GPU <-> pinned-DRAM moves ran as fused-kernel launches (digest on the tensor cores), not staged memcpys
        assert r["fused_tier_moves"] >= 3 and r["promoted_back"], r
    finally:
        cl.stop()


def test_tile_trace_records_the_pipeline(bb, torch_cuda):
    """Diagnostics (SURVEY 5.1): per-tile globaltimer stamps of the fused kernel's producer and store warps."""
    torch = torch_cuda
    import numpy as np

    eng = bb.XferEngine(0, 64, 2)
    n = 8 << 20
    src = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda")
    dst = torch.zeros_like(src)
    eng.set_tile_trace(True)
    dg, st, _ = eng.run([(src.data_ptr(), dst.data_ptr(), n)], bb.ChecksumAlgo.BBH64, _stream(torch))
    torch.cuda.synchronize()
    assert st == [0] and torch.equal(src, dst)
    t = np.asarray(eng.tile_trace(), dtype=np.uint64).reshape(-1, 4).astype(np.int64)
    assert t.shape[0] == n // 16384 and (t > 0).all()
    assert (t[:, 1] >= t[:, 0]).all() and (t[:, 2] >= t[:, 1]).all() and (t[:, 3] >= t[:, 2]).all()  # issue <= landed <= stored <= released
    eng.set_tile_trace(False)
    eng.run([(src.data_ptr(), dst.data_ptr(), n)], bb.ChecksumAlgo.BBH64, _stream(torch))


def test_tensor_store_fused_fp8_path(bb, torch_cuda):
    """TensorStore.put(pack_fp8=True) on whole-tile bf16 tensors uses the fused pack-put / unpack-get kernels; the stored
    object is the same MXFP8 object the unfused path writes (a plain device get + mxfp8_unpack reads it too)."""
    torch = torch_cuda
    from blackbird_b200.ops import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id="t-fp8")
    try:
        ts = TensorStore(cl.client)
        kv = (torch.randn(8, 16384, device="cuda") * 2).to(torch.bfloat16)  # 8 tiles
        odd = (torch.randn(1000, 33, device="cuda")).to(torch.bfloat16)     # not tile aligned -> unfused path
        l0 = cl.fabric.launches
        ts.batch_put(["kv", "odd"], [kv, odd], pack_fp8=True)
        sh = cl.client.get_workers("kv")[0].shards[0]
        n = kv.numel()
        assert sh.length == n + n // 32 and sh.checksum_algo == bb.ChecksumAlgo.BBH64
        raw = torch.empty(sh.length, dtype=torch.uint8, device="cuda")
        ecs, _ = cl.client.batch_get_device(["kv"], [raw.data_ptr()], [sh.length], _stream(torch))  # plain verified get of the packed bytes
        assert ecs == [bb.ErrorCode.OK]
        ref = torch.empty_like(raw)
        bb.mxfp8_pack(kv.data_ptr(), n, ref.data_ptr(), _stream(torch))
        torch.cuda.synchronize()
        assert torch.equal(raw, ref) and sh.checksum == bb.bbh64(raw.cpu().numpy())
        back_kv, back_odd = ts.batch_get(["kv", "odd"])
        torch.cuda.synchronize()
        unp = torch.empty_like(kv)
        bb.mxfp8_unpack(ref.data_ptr(), n, unp.data_ptr(), _stream(torch))
        torch.cuda.synchronize()
        assert back_kv.shape == kv.shape and torch.equal(back_kv.view(torch.int16), unp.view(torch.int16))
        assert back_odd.shape == odd.shape and (back_odd.float() - odd.float()).abs().max().item() <= odd.float().abs().max().item() * 2 ** -3
        # corruption of the stored scales is caught by the fused get
        cl.worker.backend("hbm0").write(sh.offset + n + 3, b"\x7f")
        with pytest.raises(RuntimeError):
            ts.get("kv")
        assert cl.fabric.launches - l0 >= 6
    finally:
        cl.stop()


def test_async_tensor_store_overlaps_and_local_replica_is_preferred(bb, torch_cuda):
    """AsyncTensorStore: transfers run on a side stream from a worker thread (futures), ordered after the producer's
    stream; a get whose replica lives on the client's own GPU is served from it (no fabric hop)."""
    torch = torch_cuda
    from blackbird_b200.ops import AsyncTensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=512 << 20, cluster_id="t-async")
    try:
        ts = AsyncTensorStore(cl.client)
        a = torch.randn(2048, 2048, device="cuda")
        acts = []
        futs = []
        for i in range(4):
            a = torch.tanh(a @ a.t() / 2048.0)  # producer work on the main stream
            acts.append(a)
            futs.append(ts.put_async([f"act/{i}"], [a]))  # must observe the finished matmul (event wait)
        assert [f.result(timeout=60) for f in futs] == [1, 1, 1, 1]
        got = ts.get_async([f"act/{i}" for i in range(4)]).result(timeout=60)
        torch.cuda.synchronize()
        for g, ref in zip(got, acts):
            assert torch.equal(g, ref)
        kv = (torch.randn(4, 16384, device="cuda")).to(torch.bfloat16)
        assert ts.put_async(["kv"], [kv], pack_fp8=True).result(timeout=60) == 1
        back = ts.get_async(["kv"]).result(timeout=60)[0]
        assert back.shape == kv.shape and (back.float() - kv.float()).abs().max().item() <= kv.float().abs().max().item() * 2 ** -3
        ts.close()
        assert "bb_client_device_get_local_replica_total" in cl.client.metrics_text()
    finally:
        cl.stop()


def test_dram_tier_is_reached_by_the_fused_kernels(bb, torch_cuda):
    """Objects placed in (or demoted to) a pinned DRAM pool are moved by the SAME fused kernel over PCIe -- TMA from /
    to registered host memory, digest on the tensor cores -- not staged through the TCP data server."""
    torch = torch_cuda
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id="t-dram", dram_bytes=128 << 20)
    try:
        n, size = 8, (1 << 20) + 48
        stride = ((size + 255) // 256) * 256
        src = torch.randint(0, 256, (n * stride,), dtype=torch.uint8, device="cuda")
        out = torch.zeros_like(src)
        keys = [f"d{i}" for i in range(n)]
        cfg = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, preferred_classes=[bb.StorageClass.RAM_CPU])
        s = _stream(torch)
        l0 = cl.fabric.launches
        ecs = cl.client.batch_put_device(keys, [src.data_ptr() + i * stride for i in range(n)], [size] * n, cfg, s)
        assert all(e == bb.ErrorCode.OK for e in ecs), ecs
        assert cl.fabric.mapped_host_pools() == 1 and cl.fabric.launches == l0 + 1  # one fused launch wrote the DRAM pool
        sh = cl.client.get_workers(keys[2])[0].shards[0]
        assert sh.storage_class == bb.StorageClass.RAM_CPU and sh.location["kind"] == "memory"
        assert sh.checksum == bb.bbh64(src[2 * stride:2 * stride + size].cpu().numpy())
        ecs, sizes = cl.client.batch_get_device(keys, [out.data_ptr() + i * stride for i in range(n)], [stride] * n, s)
        assert all(e == bb.ErrorCode.OK for e in ecs) and sizes == [size] * n
        torch.cuda.synchronize()
        assert cl.fabric.launches == l0 + 2
        for i in range(n):
            assert torch.equal(src[i * stride:i * stride + size], out[i * stride:i * stride + size])
        assert "device_get_dram_direct_total" in cl.client.metrics_text()
        assert cl.fabric.path_bytes(True, 2) == n * size and cl.fabric.path_bytes(False, 2) == n * size  # over PCIe
        # the worker's own view of the pool (host path) holds the same bytes, and corruption there is caught by the fused get
        be = cl.worker.backend(f"dram{cl.rank}")
        pool = [p for p in cl.client.keystone().get_memory_pools() if p.id == sh.pool_id][0]
        off = sh.location["remote_addr"] - pool.ucx_remote_addr
        assert be.read(off, 64) == bytes(src[2 * stride:2 * stride + 64].cpu().numpy())
        be.write(off + 100, b"\xff\x00\xff\x00")
        ecs, _ = cl.client.batch_get_device([keys[2]], [out.data_ptr()], [stride], s)
        assert ecs[0] == bb.ErrorCode.CHECKSUM_MISMATCH
    finally:
        cl.stop()


def test_fused_fp8_put_fans_out_to_replicas_and_get_fails_over(bb, torch_cuda):
    """Fused MXFP8 put with replication: the tile is converted once and TMA-stored to every copy (payload + scales);
    every copy holds the bytes of the stand-alone pack kernel; a fused get whose replica is corrupt verifies the digest,
    reports the mismatch and is retried on the next replica."""
    torch = torch_cuda
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id="t-fp8r")
    try:
        s = _stream(torch)
        nobj, n = 3, 5 * 16384
        xs = [(torch.randn(n, device="cuda") * (i + 1)).to(torch.bfloat16) for i in range(nobj)]
        keys = [f"fp8r/{i}" for i in range(nobj)]
        cfg = bb.WorkerConfig(replication_factor=3, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_GPU])
        l0 = cl.fabric.launches
        ecs = cl.client.batch_put_device_fp8(keys, [x.data_ptr() for x in xs], [n] * nobj, cfg, s)
        assert ecs == [bb.ErrorCode.OK] * nobj, ecs
        assert cl.fabric.launches - l0 == 2  # pack+fan-out kernel, scales hash slice: replicas cost no extra launch
        be = cl.worker.backend("hbm0")
        for i, k in enumerate(keys):
            copies = cl.client.get_workers(k)
            assert len(copies) == 3 and len({c.shards[0].offset for c in copies}) == 3
            ref = torch.empty(n + n // 32, dtype=torch.uint8, device="cuda")
            bb.mxfp8_pack(xs[i].data_ptr(), n, ref.data_ptr(), s)
            torch.cuda.synchronize()
            ref_b = bytes(ref.cpu().numpy())
            for c in copies:
                sh = c.shards[0]
                assert sh.checksum == bb.bbh64(ref.cpu().numpy()) and be.read(sh.offset, sh.length) == ref_b
        # corrupt two of the three copies of object 1: the get must end on the intact one
        copies = cl.client.get_workers(keys[1])
        for c in copies[:2]:
            be.write(c.shards[0].offset + 777, b"\x01\x02\x03\x04")
        outs = [torch.zeros_like(x) for x in xs]
        ecs = cl.client.batch_get_device_fp8(keys, [o.data_ptr() for o in outs], [n] * nobj, s)
        torch.cuda.synchronize()
        assert ecs == [bb.ErrorCode.OK] * nobj, ecs
        for x, o in zip(xs, outs):
            unp = torch.empty_like(x)
            ref = torch.empty(n + n // 32, dtype=torch.uint8, device="cuda")
            bb.mxfp8_pack(x.data_ptr(), n, ref.data_ptr(), s)
            bb.mxfp8_unpack(ref.data_ptr(), n, unp.data_ptr(), s)
            torch.cuda.synchronize()
            assert torch.equal(o.view(torch.int16), unp.view(torch.int16))
        # all three corrupt -> CHECKSUM_MISMATCH (a flipped byte: writing a constant leaves a copy intact whose byte holds it)
        _flip_byte(be, copies[2].shards[0].offset + 5)
        ecs = cl.client.batch_get_device_fp8([keys[1]], [outs[1].data_ptr()], [n], s)
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH]
    finally:
        cl.stop()


def _flip_byte(be, offset):
    be.write(offset, bytes([be.read(offset, 1)[0] ^ 0xFF]))


def test_device_get_fails_over_to_the_next_replica(bb, torch_cuda):
    """A plain device get whose replica is corrupt: the fused kernel reports the mismatch and the client re-reads the
    object from the next replica, until one verifies; with every copy corrupt the get reports CHECKSUM_MISMATCH."""
    torch = torch_cuda
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id="t-failover")
    try:
        s = _stream(torch)
        n, size = 4, 100000
        stride = ((size + 255) // 256) * 256
        src = torch.randint(0, 256, (n * stride,), dtype=torch.uint8, device="cuda")
        keys = [f"fo/{i}" for i in range(n)]
        cfg = bb.WorkerConfig(replication_factor=3, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_GPU])
        ecs = cl.client.batch_put_device(keys, [src.data_ptr() + i * stride for i in range(n)], [size] * n, cfg, s)
        assert ecs == [bb.ErrorCode.OK] * n, ecs
        be = cl.worker.backend("hbm0")
        copies = cl.client.get_workers(keys[1])
        assert len(copies) == 3 and len({c.shards[0].offset for c in copies}) == 3
        # corrupt two of the three copies of object 1: the get must end on the intact one
        for c in copies[:2]:
            _flip_byte(be, c.shards[0].offset + 777)
        out = torch.zeros_like(src)
        ecs, sizes = cl.client.batch_get_device(keys, [out.data_ptr() + i * stride for i in range(n)], [stride] * n, s)
        torch.cuda.synchronize()
        assert ecs == [bb.ErrorCode.OK] * n and sizes == [size] * n, ecs
        for i in range(n):
            assert torch.equal(src[i * stride:i * stride + size], out[i * stride:i * stride + size])
        assert "bb_client_replica_failover_total" in cl.client.metrics_text()
        # all three corrupt -> CHECKSUM_MISMATCH
        _flip_byte(be, copies[2].shards[0].offset + 5)
        ecs, _ = cl.client.batch_get_device([keys[1]], [out.data_ptr() + stride], [stride], s)
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH]
    finally:
        cl.stop()


def test_device_get_of_a_batch_that_mixes_checksum_algorithms(bb, torch_cuda):
    """Objects written with XXH3 and with CRC32C, read back in one batch_get_device: each is verified against its own
    algorithm's digest, and a corrupt object in each group is reported for that object only."""
    torch = torch_cuda
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id="t-mixalgo")
    try:
        s = _stream(torch)
        sizes = [5000, 70000, 16384, 300, 100000, 4096]
        algos = [bb.ChecksumAlgo.XXH3] * 3 + [bb.ChecksumAlgo.CRC32C] * 3
        n, stride = len(sizes), 100096
        src = torch.randint(0, 256, (n * stride,), dtype=torch.uint8, device="cuda")
        keys = [f"mix/{i}" for i in range(n)]
        for i in range(n):
            cfg = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_GPU],
                                  checksum=algos[i])
            assert cl.client.batch_put_device([keys[i]], [src.data_ptr() + i * stride], [sizes[i]], cfg, s) == [bb.ErrorCode.OK]
        shards = [cl.client.get_workers(k)[0].shards[0] for k in keys]
        assert [sh.checksum_algo for sh in shards] == algos
        out = torch.zeros_like(src)
        ptrs = [out.data_ptr() + i * stride for i in range(n)]
        ecs, got = cl.client.batch_get_device(keys, ptrs, [stride] * n, s)
        torch.cuda.synchronize()
        assert ecs == [bb.ErrorCode.OK] * n and got == sizes, ecs
        for i in range(n):
            assert torch.equal(src[i * stride:i * stride + sizes[i]], out[i * stride:i * stride + sizes[i]])
        # one corrupt object per algorithm
        be = cl.worker.backend("hbm0")
        for i in (1, 4):
            _flip_byte(be, shards[i].offset + sizes[i] // 2)
        ecs, _ = cl.client.batch_get_device(keys, ptrs, [stride] * n, s)
        want = [bb.ErrorCode.CHECKSUM_MISMATCH if i in (1, 4) else bb.ErrorCode.OK for i in range(n)]
        assert ecs == want, ecs
    finally:
        cl.stop()


@pytest.mark.parametrize("n", [32, 96, 16384 + 32, 3 * 16384 + 7 * 32, 2 * 16384 + 16352, 5 * 16384])
def test_fused_fp8_handles_any_whole_number_of_mx_blocks(bb, torch_cuda, n):
    """The fused pack-put / unpack-get kernels take any multiple of 32 elements: the tail tile is converted and stored
    like the others (scale bytes past the last 16-byte multiple byte-wise) and the digest still equals BBH64 of the
    stand-alone pack kernel's output."""
    torch = torch_cuda
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id=f"t-fp8odd{n}")
    try:
        s = _stream(torch)
        x = (torch.randn(n, device="cuda") * 3).to(torch.bfloat16)
        cfg = bb.WorkerConfig(replication_factor=2, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_GPU])
        assert cl.client.device_fp8_eligible(n)
        assert cl.client.batch_put_device_fp8(["odd"], [x.data_ptr()], [n], cfg, s) == [bb.ErrorCode.OK]
        ref = torch.empty(n + n // 32, dtype=torch.uint8, device="cuda")
        bb.mxfp8_pack(x.data_ptr(), n, ref.data_ptr(), s)
        torch.cuda.synchronize()
        be = cl.worker.backend("hbm0")
        copies = cl.client.get_workers("odd")
        assert len(copies) == 2
        for c in copies:
            sh = c.shards[0]
            assert sh.length == n + n // 32 and be.read(sh.offset, sh.length) == bytes(ref.cpu().numpy())
            assert sh.checksum == bb.bbh64(ref.cpu().numpy())
        out = torch.zeros_like(x)
        guard = torch.full((64,), 7, dtype=torch.bfloat16, device="cuda")  # the get must not write past n elements
        buf = torch.cat([out, guard])
        assert cl.client.batch_get_device_fp8(["odd"], [buf.data_ptr()], [n], s) == [bb.ErrorCode.OK]
        unp = torch.empty_like(x)
        bb.mxfp8_unpack(ref.data_ptr(), n, unp.data_ptr(), s)
        torch.cuda.synchronize()
        assert torch.equal(buf[:n].view(torch.int16), unp.view(torch.int16)) and bool((buf[n:] == 7).all())
        # corruption in the tail region (payload tail or scales) is caught
        for c, pos in ((copies[0], n - 1), (copies[1], n + n // 32 - 1)):
            off = c.shards[0].offset + pos
            be.write(off, bytes([be.read(off, 1)[0] ^ 0xFF]))
        assert cl.client.batch_get_device_fp8(["odd"], [buf.data_ptr()], [n], s) == [bb.ErrorCode.CHECKSUM_MISMATCH]
    finally:
        cl.stop()


def test_pipeline_soak_random_layouts_tails_and_fanout(bb, torch_cuda):
    """Soak of the kernel's mbarrier / stage-metadata protocol (the racecheck report reasons about it; this stresses it): ~10^6
    tiles through the persistent pipeline as batches of randomly sized objects (whole tiles, tiles +- a few bytes, odd tails,
    multi-MiB objects split over CTAs) with 1-3 destinations each and a different digest every round.  A tile handled with another
    tile's metadata (stale size, destination, object index, tile index) shows up as a wrong byte, a stray write outside the
    objects, a digest that differs from the CPU model, or a verify mismatch on the read-back."""
    torch = torch_cuda
    tile = bb.TILE_BYTES
    B = 512 << 20
    eng = bb.XferEngine(0, 1 << 16, 2)
    stream = _stream(torch)
    src = torch.empty(B, dtype=torch.uint8, device="cuda")
    dsts = [torch.empty(B, dtype=torch.uint8, device="cuda") for _ in range(3)]
    back = torch.empty(B, dtype=torch.uint8, device="cuda")
    rng = np.random.default_rng(0xB200)
    algos = [("XXH3", bb.xxh3t64), ("CRC32C", bb.crc32c), ("BBH64", bb.bbh64), ("NONE", None)]
    tiles_done, rnd = 0, -1
    while tiles_done < 1_000_000:
        rnd += 1
        name, host_digest = algos[rnd % len(algos)]
        algo = getattr(bb.ChecksumAlgo, name)
        bb.random_fill(src.data_ptr(), B, 1000 + rnd, stream)
        for d in dsts:
            d.zero_()
        back.zero_()
        # layout: objects back to back at 256-byte aligned offsets
        sizes, offs, ndst, off = [], [], [], 0
        while True:
            kind = rng.integers(0, 10)
            if kind < 3:
                n = int(rng.integers(1, 12)) * tile
            elif kind < 6:
                n = max(1, int(rng.integers(1, 12)) * tile + int(rng.integers(-255, 256)))
            elif kind < 9:
                n = int(rng.integers(1, 200000))
            else:
                n = int(rng.integers(1 << 20, 8 << 20)) + int(rng.integers(0, 16))
            if off + n > B:
                break
            sizes.append(n), offs.append(off), ndst.append(int(rng.integers(1, 4)))
            off = (off + n + 255) // 256 * 256
        nobj = len(sizes)
        items = [(src.data_ptr() + o, [dsts[k].data_ptr() + o for k in range(r)], n) for o, n, r in zip(offs, sizes, ndst)]
        dg, st, _ = eng.run(items, algo, stream)
        assert not any(st)
        tiles_done += sum((n + tile - 1) // tile for n in sizes)
        t_off = torch.tensor(offs, dtype=torch.int64, device="cuda")
        t_end = t_off + torch.tensor(sizes, dtype=torch.int64, device="cuda")
        t_nd = torch.tensor(ndst, dtype=torch.int64, device="cuda")
        masks = []
        for k in range(3):
            sel = t_nd > k
            edge = torch.zeros(B + 1, dtype=torch.int8, device="cuda")
            edge[t_off[sel]] += 1
            edge[t_end[sel]] -= 1
            m = torch.cumsum(edge, 0, dtype=torch.int8)[:B] > 0
            masks.append(m)
            assert torch.equal(dsts[k][m], src[m]), f"round {rnd}: wrong bytes in destination {k}"
            assert not bool(dsts[k][~m].any()), f"round {rnd}: stray write in destination {k}"
            del edge
        if host_digest is not None:
            for i in rng.choice(nobj, size=24, replace=False):
                h = src[offs[i]:offs[i] + sizes[i]].cpu().numpy()
                assert dg[i] == host_digest(h), f"round {rnd}: digest of object {i} ({sizes[i]} B)"
        # read everything back with on-device verification; one object of the stored copy is corrupted first
        bad = int(rng.integers(0, nobj))
        pos = offs[bad] + int(rng.integers(0, sizes[bad]))
        dsts[0][pos] ^= 0x40
        items = [(dsts[0].data_ptr() + o, back.data_ptr() + o, n, int(d), bb.XFER_VERIFY) for o, n, d in zip(offs, sizes, dg)]
        dg2, st2, _ = eng.run(items, algo, stream)
        tiles_done += sum((n + tile - 1) // tile for n in sizes)
        if host_digest is not None:
            assert [i for i, s in enumerate(st2) if s] == [bad], f"round {rnd}: verify flagged {[i for i, s in enumerate(st2) if s][:8]}, corrupted {bad}"
            assert all(a == b for i, (a, b) in enumerate(zip(dg, dg2)) if i != bad)
        dsts[0][pos] ^= 0x40
        back[pos] ^= 0x40
        assert torch.equal(back[masks[0]], src[masks[0]]) and not bool(back[~masks[0]].any())
        del masks
    assert rnd >= 4  # every digest took part
