"""alloc/: PoolAllocator + RangeAllocator.  Semantics follow the reference suites
tests/allocation/test_pool_allocator.cpp (10) and test_range_allocator.cpp (24); new modes
(contiguous, symmetric, narrowing instead of failing, live free-space ranking) are tested too."""
import random
import threading

import pytest


def mkpool(bb, pid, size, sc=None, node="node-a", worker="", rkey="deadbeef", ep="127.0.0.1:12345", addr=0x1000000):
    return bb.MemoryPool(pid, size, sc if sc is not None else bb.StorageClass.RAM_CPU, node, worker, ep, addr, rkey)


# ---------------------------------------------------------------- PoolAllocator
def test_pool_init_single_free_range(bb):
    pa = bb.PoolAllocator(mkpool(bb, "p", 1 << 20))
    assert pa.total_free() == 1 << 20 and pa.largest_free_block() == 1 << 20
    assert pa.fragmentation_ratio() == 0.0 and len(pa.free_ranges()) == 1


def test_pool_exact_alloc_and_merge_back(bb):
    pa = bb.PoolAllocator(mkpool(bb, "p", 4096))
    r = pa.allocate(4096)
    assert r.offset == 0 and r.length == 4096 and pa.total_free() == 0
    assert pa.allocate(256) is None
    pa.free(r)
    assert pa.total_free() == 4096 and len(pa.free_ranges()) == 1


def test_pool_split_remainder_and_alignment(bb):
    pa = bb.PoolAllocator(mkpool(bb, "p", 8192))
    r = pa.allocate(1000)
    assert r.offset == 0 and r.length == 1024  # rounded to the 256 B extent alignment
    fr = pa.free_ranges()
    assert len(fr) == 1 and fr[0].offset == 1024 and fr[0].length == 8192 - 1024


def test_pool_best_fit_picks_tightest_hole_first_fit_lowest(bb):
    pa = bb.PoolAllocator(mkpool(bb, "p", 16384))
    a = pa.allocate(4096)
    b = pa.allocate(1024)
    c = pa.allocate(2048)
    d = pa.allocate(512)
    pa.free(a)  # hole of 4096 at 0
    pa.free(c)  # hole of 2048 at 5120
    best = pa.allocate(2048, True)
    assert best.offset == c.offset  # tightest hole
    pa.free(best)
    first = pa.allocate(2048, False)
    assert first.offset == 0  # lowest offset
    assert b.offset == 4096 and d.offset == 7168


def test_pool_coalescing_prev_next_both_none(bb):
    pa = bb.PoolAllocator(mkpool(bb, "p", 4096))
    rs = [pa.allocate(1024) for _ in range(4)]
    pa.free(rs[0])
    pa.free(rs[2])
    assert len(pa.free_ranges()) == 2  # no neighbours yet
    pa.free(rs[1])  # merges with prev and next
    fr = pa.free_ranges()
    assert len(fr) == 1 and fr[0].offset == 0 and fr[0].length == 3072
    pa.free(rs[3])
    assert len(pa.free_ranges()) == 1 and pa.largest_free_block() == 4096


def test_pool_fragmentation_ratio_formula(bb):
    pa = bb.PoolAllocator(mkpool(bb, "p", 4096))
    rs = [pa.allocate(1024) for _ in range(4)]
    pa.free(rs[0])
    pa.free(rs[2])
    assert pa.total_free() == 2048 and pa.largest_free_block() == 1024
    assert abs(pa.fragmentation_ratio() - 0.5) < 1e-9  # 1 - largest/total


def test_pool_allocate_at_and_double_free_is_rejected(bb):
    pa = bb.PoolAllocator(mkpool(bb, "p", 8192))
    assert pa.allocate_at(2048, 1024)
    assert not pa.allocate_at(2048, 256)  # taken
    assert not pa.allocate_at(100, 256)   # misaligned
    assert pa.total_free() == 8192 - 1024
    pa.free(bb.Range(2048, 1024))
    pa.free(bb.Range(2048, 1024))  # logged, ignored
    assert pa.total_free() == 8192


def test_pool_concurrent_alloc_until_full_then_shuffled_free(bb):
    pa = bb.PoolAllocator(mkpool(bb, "p", 1 << 20))
    got = [[] for _ in range(8)]

    def worker(i):
        while True:
            r = pa.allocate(1024)
            if r is None:
                return
            got[i].append(r)

    ts = [threading.Thread(target=worker, args=(i,)) for i in range(8)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    allr = [r for g in got for r in g]
    assert len(allr) == 1024 and len({r.offset for r in allr}) == 1024 and pa.total_free() == 0
    random.Random(1).shuffle(allr)
    chunks = [allr[i::8] for i in range(8)]
    ts = [threading.Thread(target=lambda c=c: [pa.free(r) for r in c]) for c in chunks]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert pa.total_free() == 1 << 20 and len(pa.free_ranges()) == 1  # fully coalesced


# ---------------------------------------------------------------- RangeAllocator
def req(bb, key, size, repl=1, wpc=1, classes=None, node="", min_shard=4096, **kw):
    return bb.AllocationRequest(key, size, repl, wpc, classes if classes is not None else [bb.StorageClass.RAM_CPU], node,
                                min_shard_size=min_shard, **kw)


def test_range_empty_stats_and_empty_pool_map(bb):
    ra = bb.RangeAllocator()
    st = ra.get_stats()
    assert st.total_objects == 0 and st.total_shards == 0 and st.total_allocated_bytes == 0
    with pytest.raises(bb.BlackbirdError) as e:
        ra.allocate(req(bb, "k", 1024), {})
    assert e.value.code == bb.ErrorCode.INSUFFICIENT_SPACE


def test_range_can_allocate_class_filter(bb):
    ra = bb.RangeAllocator()
    pools = {"p1": mkpool(bb, "p1", 1 << 20, bb.StorageClass.RAM_CPU)}
    assert ra.can_allocate(req(bb, "k", 4096, classes=[bb.StorageClass.RAM_CPU]), pools)
    assert not ra.can_allocate(req(bb, "k", 4096, classes=[bb.StorageClass.NVME]), pools)
    assert not ra.can_allocate(req(bb, "k", 2 << 20), pools)


def test_range_two_way_striping_with_endpoint_rkey_addr(bb):
    ra = bb.RangeAllocator()
    pools = {"p1": mkpool(bb, "p1", 1 << 20, addr=0x10000000), "p2": mkpool(bb, "p2", 1 << 20, addr=0x20000000, rkey="cafebabe")}
    res = ra.allocate(req(bb, "obj", 16384, wpc=2), pools)
    assert len(res.copies) == 1 and len(res.copies[0].shards) == 2 and res.total_shards_created == 2 and res.pools_used == 2
    shards = res.copies[0].shards
    assert {s.pool_id for s in shards} == {"p1", "p2"} and sum(s.length for s in shards) == 16384
    for s in shards:
        assert s.length == 8192 and s.endpoint.ip == "127.0.0.1" and s.endpoint.port == 12345
        loc = s.location
        assert loc["kind"] == "memory" and loc["size"] == 8192
        base = 0x10000000 if s.pool_id == "p1" else 0x20000000
        assert loc["remote_addr"] >= base and loc["rkey"] == (0xDEADBEEF if s.pool_id == "p1" else 0xCAFEBABE)
        assert s.endpoint.worker_key == bytes.fromhex("deadbeef" if s.pool_id == "p1" else "cafebabe")


def test_range_three_replicas_two_shards_over_six_pools(bb):
    ra = bb.RangeAllocator()
    pools = {f"p{i}": mkpool(bb, f"p{i}", 1 << 20) for i in range(6)}
    res = ra.allocate(req(bb, "obj", 32768, repl=3, wpc=2), pools)
    assert len(res.copies) == 3 and all(len(c.shards) == 2 for c in res.copies)
    used = [s.pool_id for c in res.copies for s in c.shards]
    assert len(set(used)) == 6  # every replica shard on its own pool
    assert [c.copy_index for c in res.copies] == [0, 1, 2]


def test_range_min_shard_strict_fails_default_narrows(bb):
    pools = {f"p{i}": mkpool(bb, f"p{i}", 8192) for i in range(4)}
    ra = bb.RangeAllocator()
    with pytest.raises(bb.BlackbirdError) as e:  # reference semantics
        ra.allocate(req(bb, "small", 1024, wpc=4, min_shard=4096, strict_min_shard=True), pools)
    assert e.value.code == bb.ErrorCode.INSUFFICIENT_SPACE
    res = ra.allocate(req(bb, "small", 1024, wpc=4, min_shard=4096), pools)  # GPU store: narrow the stripe
    assert len(res.copies[0].shards) == 1 and res.copies[0].shards[0].length == 1024
    pools8 = {f"q{i}": mkpool(bb, f"q{i}", 16384) for i in range(8)}
    with pytest.raises(bb.BlackbirdError):
        bb.RangeAllocator().allocate(req(bb, "x", 4096, wpc=8, min_shard=2048, strict_min_shard=True), pools8)
    res = bb.RangeAllocator().allocate(req(bb, "x", 4096, wpc=8, min_shard=2048), pools8)
    assert len(res.copies[0].shards) == 2


def test_range_insufficient_capacity_and_rollback(bb):
    ra = bb.RangeAllocator()
    pools = {"p1": mkpool(bb, "p1", 4096), "p2": mkpool(bb, "p2", 4096)}
    with pytest.raises(bb.BlackbirdError) as e:
        ra.allocate(req(bb, "big", 16384, wpc=2), pools)
    assert e.value.code == bb.ErrorCode.INSUFFICIENT_SPACE
    # nothing leaked: the full capacity is still allocatable
    res = ra.allocate(req(bb, "fits", 8192, wpc=2), pools)
    assert sum(s.length for s in res.copies[0].shards) == 8192
    assert ra.get_stats().total_objects == 1


def test_range_class_preference_and_spillover_fallback(bb):
    ra = bb.RangeAllocator()
    pools = {"ram": mkpool(bb, "ram", 8192, bb.StorageClass.RAM_CPU), "nvme": mkpool(bb, "nvme", 1 << 20, bb.StorageClass.NVME)}
    res = ra.allocate(req(bb, "a", 4096, classes=[bb.StorageClass.RAM_CPU]), pools)
    assert res.copies[0].shards[0].pool_id == "ram" and not res.required_spillover
    res = ra.allocate(req(bb, "b", 65536, classes=[bb.StorageClass.RAM_CPU]), pools)  # does not fit in RAM
    assert res.copies[0].shards[0].pool_id == "nvme" and res.required_spillover
    assert res.copies[0].shards[0].location["kind"] == "file"


def test_range_uneven_split_1000_by_3(bb):
    ra = bb.RangeAllocator()
    pools = {f"p{i}": mkpool(bb, f"p{i}", 1 << 16) for i in range(3)}
    res = ra.allocate(req(bb, "odd", 1000, wpc=3, min_shard=1), pools)
    assert [s.length for s in res.copies[0].shards] == [334, 333, 333]


def test_range_replication_stress_5x_and_20x(bb):
    for repl in (5, 20):
        ra = bb.RangeAllocator()
        pools = {f"p{i}": mkpool(bb, f"p{i}", 1 << 20) for i in range(repl)}
        res = ra.allocate(req(bb, "r", 8192, repl=repl, wpc=1), pools)
        assert len(res.copies) == repl
        assert len({c.shards[0].pool_id for c in res.copies}) == repl  # one replica per pool


def test_range_malformed_endpoint_or_rkey_is_invalid_parameters(bb):
    for bad in (dict(ep="not-an-endpoint"), dict(ep="host:notaport"), dict(rkey="xyz")):
        ra = bb.RangeAllocator()
        with pytest.raises(bb.BlackbirdError) as e:
            ra.allocate(req(bb, "k", 4096), {"p": mkpool(bb, "p", 1 << 20, **bad)})
        assert e.value.code == bb.ErrorCode.INVALID_PARAMETERS


def test_range_fragmentation_then_merged_realloc(bb):
    ra = bb.RangeAllocator()
    pools = {"p": mkpool(bb, "p", 8192)}
    for i in range(8):
        ra.allocate(req(bb, f"o{i}", 1024), pools)
    with pytest.raises(bb.BlackbirdError):
        ra.allocate(req(bb, "more", 1024), pools)
    for i in (1, 2, 3):
        assert ra.free(f"o{i}") == bb.ErrorCode.OK
    res = ra.allocate(req(bb, "merged", 3072), pools)  # needs the three freed extents coalesced
    assert res.copies[0].shards[0].length == 3072


def test_range_zero_size_is_tolerated(bb):
    ra = bb.RangeAllocator()
    res = ra.allocate(req(bb, "zero", 0), {"p": mkpool(bb, "p", 8192)})
    assert len(res.copies) == 1 and all(s.length == 0 for s in res.copies[0].shards)
    assert ra.free("zero") == bb.ErrorCode.OK


def test_range_preferred_node_honoured(bb):
    ra = bb.RangeAllocator()
    pools = {"a": mkpool(bb, "a", 1 << 20, node="node-a"), "b": mkpool(bb, "b", 1 << 20, node="node-b")}
    for _ in range(4):
        res = ra.allocate(req(bb, f"k{_}", 4096, node="node-b"), pools)
        assert res.copies[0].shards[0].pool_id == "b"
    with pytest.raises(bb.BlackbirdError):
        ra.allocate(req(bb, "nowhere", 4096, node="node-z"), pools)


def test_range_duplicate_key_and_realloc_after_free(bb):
    ra = bb.RangeAllocator()
    pools = {"p": mkpool(bb, "p", 1 << 20)}
    ra.allocate(req(bb, "dup", 4096), pools)
    with pytest.raises(bb.BlackbirdError) as e:
        ra.allocate(req(bb, "dup", 4096), pools)
    assert e.value.code == bb.ErrorCode.OBJECT_ALREADY_EXISTS
    assert ra.free("dup") == bb.ErrorCode.OK
    ra.allocate(req(bb, "dup", 4096), pools)
    assert ra.free("unknown") == bb.ErrorCode.OBJECT_NOT_FOUND


def test_range_64k_over_16_of_20_pools_distinct_addresses(bb):
    ra = bb.RangeAllocator()
    pools = {f"p{i:02d}": mkpool(bb, f"p{i:02d}", 1 << 20, addr=0x1000000 * (i + 1)) for i in range(20)}
    res = ra.allocate(req(bb, "wide", 65536, wpc=16), pools)
    shards = res.copies[0].shards
    assert len(shards) == 16 and len({s.pool_id for s in shards}) == 16 and all(s.length == 4096 for s in shards)
    for s in shards:
        assert s.location["remote_addr"] >= pools[s.pool_id].ucx_remote_addr
    res2 = ra.allocate(req(bb, "wide2", 65536, wpc=16), pools)
    spans = [(s.pool_id, s.location["remote_addr"]) for r in (res, res2) for s in r.copies[0].shards]
    assert len(set(spans)) == 32  # no overlap between objects


def test_range_contiguous_is_implemented_and_wpc1_works(bb):
    ra = bb.RangeAllocator()
    pools = {f"p{i}": mkpool(bb, f"p{i}", 1 << 20) for i in range(4)}
    res = ra.allocate(req(bb, "c", 1 << 18, wpc=4, prefer_contiguous=True), pools)
    assert len(res.copies[0].shards) == 1  # reference: NOT_IMPLEMENTED (range_allocator.cpp:412-417)
    res = ra.allocate(req(bb, "c1", 1 << 18, wpc=1), pools)  # the reference's default client config fails here
    assert len(res.copies[0].shards) == 1


def test_range_live_free_space_ranking_balances_pools(bb):
    """Bug #3 of the reference: ranking used the registration snapshot, so one pool filled up first."""
    ra = bb.RangeAllocator()
    pools = {f"p{i}": mkpool(bb, f"p{i}", 1 << 20) for i in range(4)}
    for i in range(64):
        ra.allocate(req(bb, f"o{i}", 8192), pools)
    used = [ra.pool_used_bytes(f"p{i}") for i in range(4)]
    assert max(used) - min(used) <= 8192


def test_range_replicas_prefer_distinct_workers(bb):
    ra = bb.RangeAllocator()
    pools = {}
    for w in range(3):
        for k in range(2):
            pools[f"w{w}p{k}"] = mkpool(bb, f"w{w}p{k}", 1 << 20, worker=f"worker-{w}")
    res = ra.allocate(req(bb, "r3", 16384, repl=3, wpc=1), pools)
    workers = {pools[c.shards[0].pool_id].worker_id for c in res.copies}
    assert len(workers) == 3  # one replica per failure domain


def test_range_symmetric_replicas_share_one_offset(bb):
    ra = bb.RangeAllocator()
    G = bb.StorageClass.RAM_GPU
    pools = {f"g{i}": bb.MemoryPool(f"g{i}", 1 << 20, G, f"gpu{i}", f"w{i}", "127.0.0.1:1", 0, "00", i) for i in range(4)}
    ra.allocate(req(bb, "skew", 4096, classes=[G], node="gpu1"), pools)  # make g1's free list differ
    res = ra.allocate(req(bb, "sym", 65536, repl=3, wpc=1, classes=[G], symmetric_replicas=True), pools)
    offs = {c.shards[0].location["offset"] for c in res.copies}
    assert len(res.copies) == 3 and len(offs) == 1 and all(c.shards[0].location["kind"] == "gpu" for c in res.copies)
    assert len({c.shards[0].location["device_rank"] for c in res.copies}) == 3
    assert ra.free("sym") == bb.ErrorCode.OK


def test_range_locality_prefers_writer_node_then_fabric(bb):
    ra = bb.RangeAllocator()
    G = bb.StorageClass.RAM_GPU
    pools = {"far": bb.MemoryPool("far", 1 << 24, G, "gpu7", "w7", "127.0.0.1:1", 0, "00", 7, 0.0, "other"),
             "near": bb.MemoryPool("near", 1 << 20, G, "gpu1", "w1", "127.0.0.1:1", 0, "00", 1, 0.0, "nvswitch-0"),
             "self": bb.MemoryPool("self", 1 << 20, G, "gpu0", "w0", "127.0.0.1:1", 0, "00", 0, 0.0, "nvswitch-0")}
    r = ra.allocate(req(bb, "a", 4096, classes=[G], client_node="gpu0"), pools)
    assert r.copies[0].shards[0].pool_id == "self"
    r = ra.allocate(req(bb, "b", 4096, classes=[G], client_node="gpu0", enable_locality_awareness=False), pools)
    assert r.copies[0].shards[0].pool_id == "far"  # most free space wins without locality


def test_range_forget_pool_drops_extents_so_a_reregistered_pool_is_not_double_allocated(bb):
    """ADVICE r1 (high): worker death -> same pool id re-registered -> remove of a degraded object must not return the
    dead incarnation's offsets to the new allocator (B and C used to receive the same range)."""
    ra = bb.RangeAllocator()
    pools = {"p1": mkpool(bb, "p1", 1 << 20, worker="w1"), "p2": mkpool(bb, "p2", 1 << 20, worker="w2")}
    a = ra.allocate(req(bb, "A", 65536, repl=2, wpc=1), pools)
    assert {c.shards[0].pool_id for c in a.copies} == {"p1", "p2"}
    ra.forget_pool("p1")
    assert ra.pool_used_bytes("p1") == 0
    b = ra.allocate(req(bb, "B", 65536, repl=1, wpc=1, node="node-a"), {"p1": pools["p1"]})
    assert ra.free("A") == bb.ErrorCode.OK  # only the surviving p2 extent goes back
    c = ra.allocate(req(bb, "C", 65536, repl=1, wpc=1), {"p1": pools["p1"]})
    off = lambda r: r.copies[0].shards[0].location["remote_addr"]
    assert off(b) != off(c), "live object's range handed out twice"
    assert ra.pool_used_bytes("p1") == 2 * 65536 and ra.pool_used_bytes("p2") == 0
