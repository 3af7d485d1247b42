"""The batched transfer kernels (bb_xfer, bb_xfer_small, bb_xfer_fp8) against the CPU models, bit for bit, at the grid
sizes, batch shapes and object edges where their cross-CTA, slice and batch logic changes.  Every check reads back the
digests, the verify status, the destination bytes and the guard bytes past every object and in every gap between objects."""
import numpy as np
import pytest
import torch

from test_mxfp8 import check_packed, check_unpacked, special_blocks

pytestmark = pytest.mark.gpu

T = 16384  # bytes per tile
GUARD = 0xA5
M64 = (1 << 64) - 1
ALGOS = ["NONE", "CRC32C", "BBH64", "XXH3"]
# persistent CTAs of the kernels (XferEngine.set_max_ctas); the SM-relative ones are resolved on the device
GRIDS = [1, 2, 3, 7, 31, 127, 128, "sms", "sms+1", "2sms"]


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
    """The module's engine, back at its defaults after every test."""
    yield _engine
    _engine.set_max_ctas(0)
    _engine.set_small_path(True)
    _engine.set_mailbox(True)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _grid(g):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return {"sms": sms, "sms+1": sms + 1, "2sms": 2 * sms}.get(g, g)


def _model(bb, algo):
    """CPU model of a whole object's digest under `algo` (NONE: the engine reports 0)."""
    return {"NONE": lambda b: 0, "CRC32C": bb.crc32c, "BBH64": bb.bbh64, "XXH3": bb.xxh3t64}[algo]


class Layout:
    """Objects of the given sizes in one buffer at 16-byte aligned offsets, 16 to 31 guard bytes after each one.  Every
    buffer of a test (source, destinations, read-back) uses the same layout."""

    def __init__(self, sizes):
        self.sizes = list(sizes)
        self.offs = []
        o = 0
        for n in self.sizes:
            self.offs.append(o)
            o = (o + n + 16 + 15) & ~15
        self.total = o
        mask = np.zeros(self.total, dtype=bool)
        for o, n in zip(self.offs, self.sizes):
            mask[o:o + n] = True
        self.mask = torch.from_numpy(mask).cuda()

    def random(self, bb, seed):
        t = torch.empty(self.total, dtype=torch.uint8, device="cuda")
        bb.random_fill(t.data_ptr(), self.total, seed, _stream())
        return t

    def guarded(self):
        return torch.full((self.total,), GUARD, dtype=torch.uint8, device="cuda")

    def objects(self, host):
        return [host[o:o + n] for o, n in zip(self.offs, self.sizes)]

    def check(self, dst, src, what):
        """dst holds src's bytes inside the objects and GUARD everywhere else."""
        want = torch.where(self.mask, src, torch.full_like(src, GUARD))
        if not torch.equal(dst, want):
            pytest.fail(f"{what}: bytes differ at offsets {(dst != want).nonzero().flatten()[:8].tolist()}")


def _grid_layout(G):
    """Tile intervals [start, end) of the objects of a batch for a grid of G CTAs, and tiles per CTA run (tpc).

    G >= 4: the runs are tpc tiles, the last CTA gets none and the one before it a short run.  Object edges fall on a run
    edge, one tile after it and one tile before it, in turn; the first object spans three CTAs and the fourth run holds
    tpc one-tile objects.  G < 4: a five-tile object, a three-tile one and seven one-tile objects inside the first run."""
    if G < 4:
        tpc = 16
        total = G * tpc
        cuts = {5} | set(range(tpc - 8, tpc)) | {k * tpc + (0, 1, -1)[k % 3] for k in range(1, G)}
    else:
        tpc = min(8 if G <= 31 else 4, G - 2)
        total = G * tpc - tpc - 1
        cuts = {k * tpc + (0, 1, -1)[k % 3] for k in range(3, G)} | set(range(3 * tpc, 4 * tpc + 1))
    assert -(-total // G) == tpc  # cta_tile_run: ceil(total / G) tiles per CTA
    edges = [0] + sorted(c for c in cuts if 0 < c < total) + [total]
    return list(zip(edges[:-1], edges[1:])), tpc


TAILS = [T, 1, 15, 16, 17, T - 1, 4096, 100]  # bytes in an object's last tile, in turn


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("algo", ALGOS)
def test_bb_xfer_grid_sweep(bb, eng, algo, grid):
    """bb_xfer at grids from 1 CTA to twice the SM count (CTAs never wait for each other; cross-CTA state is atomics and a
    last-arriver test): the CRC32C shift and XOR combine, the tile-sum atomics, the in-CTA finalisation, the CRC chain
    state and the XXH3 four-tile finalizer all meet object edges on, before and after CTA-run edges."""
    G = _grid(grid)
    spans, tpc = _grid_layout(G)
    sizes = [(e - s - 1) * T + TAILS[i % len(TAILS)] for i, (s, e) in enumerate(spans)]
    lay = Layout(sizes)
    ndst = 1 + G % 3
    src = lay.random(bb, seed=G * 7 + ALGOS.index(algo))
    dsts = [lay.guarded() for _ in range(ndst)]
    eng.set_max_ctas(G)
    model = _model(bb, algo)
    a = getattr(bb.ChecksumAlgo, algo)
    items = [(src.data_ptr() + o, [d.data_ptr() + o for d in dsts], n) for o, n in zip(lay.offs, sizes)]
    dg, st, _ = eng.run(items, a, _stream())
    torch.cuda.synchronize()
    want = [model(b) for b in lay.objects(src.cpu().numpy())]
    assert list(dg) == want and list(st) == [0] * len(sizes)
    for r, d in enumerate(dsts):
        lay.check(d, src, f"destination {r}")
    # corrupt the first object (spanning CTAs) in the first tile of the second CTA run, and the last byte of the last object
    # (in the short run); read everything back with verify: exactly those two are flagged
    first = min(tpc, spans[0][1] - spans[0][0] - 1) * T + 777
    bad = [lay.offs[0] + first, lay.offs[-1] + sizes[-1] - 1]
    for o in bad:
        dsts[0][o] ^= 0x20
    out = lay.guarded()
    gets = [(dsts[0].data_ptr() + o, out.data_ptr() + o, n, w, bb.XFER_VERIFY) for o, n, w in zip(lay.offs, sizes, want)]
    dg2, st2, _ = eng.run(gets, a, _stream())
    torch.cuda.synchronize()
    lay.check(out, dsts[0], "read-back")
    assert list(dg2) == [model(b) for b in lay.objects(dsts[0].cpu().numpy())]
    flagged = [0] * len(sizes) if algo == "NONE" else [1] + [0] * (len(sizes) - 2) + [1]  # NONE verifies nothing
    assert list(st2) == flagged


FP8_SIZES = [32, T + 32, 96, 3 * T + 7 * 32, T, 2 * T]  # elements; whole-tile objects and objects ending in a partial tile


@pytest.mark.parametrize("grid", GRIDS)
def test_bb_xfer_fp8_grid_sweep(bb, eng, grid):
    """bb_xfer_fp8 put (pack) and get (unpack) at every grid: stored bytes equal mxfp8_pack_ref in every replica, the
    digest is bbh64 of the stored object, the get returns mxfp8_unpack_ref of it bit for bit.  Special-value blocks sit at
    the start of a tile, at its end and in a tail tile."""
    G = _grid(grid)
    sizes = list(FP8_SIZES)
    while sum(-(-n // T) for n in sizes) < 2 * G:  # enough tiles that every CTA gets about two
        sizes.append((len(sizes) % 4 + 2) * T + (len(sizes) % 2) * 64)
    starts = [int(v) for v in np.cumsum([0] + sizes)]  # the objects' first elements in one bf16 tensor
    N = starts[-1]
    g = torch.Generator(device="cuda").manual_seed(G)
    x = (torch.randn(N, device="cuda", generator=g) * 10 ** torch.empty(N, device="cuda").uniform_(-4, 3, generator=g)).to(torch.bfloat16)
    d = starts[3]  # object 3: three whole tiles and a 7-block tail
    x[d + T:d + T + 256] = special_blocks()                  # start of tile 1
    x[d + 3 * T - 256:d + 3 * T] = special_blocks()          # end of tile 2
    x[d + 3 * T:d + 3 * T + 224] = special_blocks(slice(1, 8))  # the tail tile
    x[starts[2] - 32:starts[2]] = special_blocks([4])        # object 1's one-block tail, whose scale is 0
    lay = Layout([bb.mxfp8_packed_bytes(n) for n in sizes])
    reps = [lay.guarded() for _ in range(1 + G % 3)]
    eng.set_max_ctas(G)
    dg, st, _ = eng.run_fp8([(x.data_ptr() + 2 * e, [r.data_ptr() + o for r in reps], n) for e, o, n in zip(starts, lay.offs, sizes)],
                            False, _stream())
    out_lay = Layout([2 * n for n in sizes])
    out = out_lay.guarded()
    dg2, st2, _ = eng.run_fp8([(out.data_ptr() + o, reps[0].data_ptr() + p, n, w) for o, p, n, w in zip(out_lay.offs, lay.offs, sizes, dg)],
                              True, _stream())
    torch.cuda.synchronize()
    stored = reps[0].cpu().numpy()
    objs = lay.objects(stored)
    assert list(dg) == [bb.bbh64(b) for b in objs]
    assert list(dg2) == list(dg) and list(st) == list(st2) == [0] * len(sizes)
    for r in reps:
        lay.check(r, reps[0], "replica")  # every replica identical, nothing written outside the objects
    # all objects as one packed array [payloads | scales] (blocks never straddle objects)
    packed = np.concatenate([b[:n] for b, n in zip(objs, sizes)] + [b[n:] for b, n in zip(objs, sizes)])
    check_packed(packed, np.frombuffer(bb.mxfp8_pack_ref(x.cpu().view(torch.int16).numpy()), dtype=np.uint8), N)
    back = out.cpu().numpy()
    assert bool((back[~out_lay.mask.cpu().numpy()] == GUARD).all()), "the get wrote outside the objects"
    back = torch.from_numpy(np.concatenate(out_lay.objects(back))).view(torch.bfloat16)
    check_unpacked(bb, back, packed, N)


@pytest.mark.parametrize("ctas", [1, 3, 0])
@pytest.mark.parametrize("algo", ["BBH64", "XXH3"])
def test_raw_sum_slices_and_hash_only_descriptors(bb, eng, algo, ctas):
    """XFER_RAW_SUM slices with a tile base: hash-only (no destination) and stored ones, mixed with whole objects in one
    batch.  Each slice is the CPU partial sum of its tiles; the slices of a partition finalise to the object's digest."""
    n = 7 * T + 1234
    partial = bb.bbh64_partial if algo == "BBH64" else bb.xxh3t64_partial
    whole = _model(bb, algo)
    # (start, end, stored): a partition of the object (only its last slice ends inside a tile), then slices that end
    # inside a tile in the middle of the object, an empty slice and a stored slice
    partition = [(0, T), (T, 4 * T), (4 * T, n)]
    extra = [(2 * T, 3 * T + 100), (5 * T, 5 * T + 17), (6 * T, 6 * T), (3 * T, 5 * T + 4000)]
    slices = partition + extra
    stored_slice = len(slices) - 1
    lay = Layout([n, 3 * T + 5, 100])  # the object, and two whole objects stored in the same batch
    src = lay.random(bb, seed=5 + ctas)
    dst = lay.guarded()
    base = src.data_ptr() + lay.offs[0]
    items = [(base + s, [dst.data_ptr() + lay.offs[0] + s] if i == stored_slice else [], e - s, 0, bb.XFER_RAW_SUM, s // T)
             for i, (s, e) in enumerate(slices)]
    items += [(src.data_ptr() + lay.offs[k], dst.data_ptr() + lay.offs[k], lay.sizes[k]) for k in (1, 2)]
    eng.set_max_ctas(ctas)
    dg, st, _ = eng.run(items, getattr(bb.ChecksumAlgo, algo), _stream())
    torch.cuda.synchronize()
    host = src.cpu().numpy()
    obj, others = lay.objects(host)[0], lay.objects(host)[1:]
    for i, (s, e) in enumerate(slices):
        # the object cut at the slice's end: the kernel zero-pads the slice's last tile
        assert dg[i] == partial(obj[:e], s // T, -(-(e - s) // T)), f"slice {i} [{s}, {e})"
    assert bb.bbh64_finalize(sum(dg[:len(partition)]) & M64, n) == whole(obj)
    assert list(dg[len(slices):]) == [whole(b) for b in others] and list(st) == [0] * len(items)
    s, e = slices[stored_slice]
    want = torch.full_like(dst, GUARD)
    want[lay.offs[0] + s:lay.offs[0] + e] = src[lay.offs[0] + s:lay.offs[0] + e]
    for k in (1, 2):
        want[lay.offs[k]:lay.offs[k] + lay.sizes[k]] = src[lay.offs[k]:lay.offs[k] + lay.sizes[k]]
    assert torch.equal(dst, want), "a hash-only slice stored bytes, or a stored one did not"


@pytest.mark.parametrize("path", ["warp", "tma", "mixed"])
@pytest.mark.parametrize("algo", ALGOS)
def test_batch_shape_boundaries(bb, eng, algo, path):
    """Batches of 1, 8, 9, 64, 65 and 300 objects (descriptors in the kernel parameters up to 8, results straight into
    pinned memory up to 64) through the warp-per-object kernel, the TMA kernel forced by set_small_path(False), and the
    TMA kernel chosen because one object is over 4096 bytes.  Zero-length items between the others report the digest of
    b"" and, with XFER_VERIFY, status 1 when their expected digest is wrong."""
    model = _model(bb, algo)
    a = getattr(bb.ChecksumAlgo, algo)
    empty = model(b"")
    eng.set_mailbox(False)  # the resident-warp mailbox has a test of its own
    eng.set_small_path(path != "tma")
    rng = np.random.default_rng(ALGOS.index(algo))
    for count in [1, 8, 9, 64, 65, 300]:
        sizes = [int(v) for v in rng.integers(1, 4097, count)]
        sizes[0] = [1, 15, 16, 17, 4096][count % 5]
        if path == "mixed":
            sizes[count // 2] = 4097 + count * 100
        ndst = 1 + count % 2
        lay = Layout(sizes)
        src = lay.random(bb, seed=count)
        dsts = [lay.guarded() for _ in range(ndst)]
        items = [(src.data_ptr() + o, [d.data_ptr() + o for d in dsts], n) for o, n in zip(lay.offs, sizes)]
        zero = list(range(0, len(items) + 1, 5))  # positions of the zero-length items in the batch
        for z in zero:
            items.insert(z, (src.data_ptr(), dsts[0].data_ptr(), 0))
        launches, small = eng.launches, eng.small_launches
        dg, st, _ = eng.run(items, a, _stream())
        torch.cuda.synchronize()
        assert eng.launches == launches + 1
        assert eng.small_launches == small + (path == "warp"), "the batch ran on the other kernel"
        want = iter(model(b) for b in lay.objects(src.cpu().numpy()))
        expect = [empty if i in zero else next(want) for i in range(len(items))]
        assert list(dg) == expect, count
        assert list(st) == [0] * len(items), count
        for d in dsts:
            lay.check(d, src, f"{count} objects")
        # read back with verify: every 7th object and every other zero-length item expect a wrong digest
        out = lay.guarded()
        wrong = {i for i in range(len(items)) if (i in zero and zero.index(i) % 2 == 1) or (i not in zero and i % 7 == 3)}
        gets, k = [], 0
        for i, it in enumerate(items):
            w = expect[i] ^ 1 if i in wrong else expect[i]
            if i in zero:
                gets.append((dsts[-1].data_ptr(), out.data_ptr(), 0, w, bb.XFER_VERIFY))
            else:
                gets.append((dsts[-1].data_ptr() + lay.offs[k], out.data_ptr() + lay.offs[k], sizes[k], w, bb.XFER_VERIFY))
                k += 1
        dg2, st2, _ = eng.run(gets, a, _stream())
        torch.cuda.synchronize()
        lay.check(out, src, f"{count} objects read back")
        assert list(dg2) == expect, count
        flagged = [int(algo != "NONE" and i in wrong) for i in range(len(items))]  # NONE verifies nothing
        zflag = [flagged[i] for i in zero]
        assert [st2[i] for i in zero] == zflag, f"{count} objects: status of the zero-length items"
        assert list(st2) == flagged, count


def test_slots_in_flight_and_their_reuse(bb):
    """All slots submitted before any wait (two streams, four algorithms, one verify mismatch), waited on in reverse order;
    then BBH64, XXH3 and CRC32C batches back to back on the same slots, every order of the three on every slot.  Objects
    span CTA runs, so each batch leaves the workspace (sum_ws: XOR for CRC32C, add for the tile sums; done_ws) behind: it
    must be zero again whatever the slot ran before."""
    slots = 4
    eng = bb.XferEngine(0, 256, slots)
    sizes = [37 * T + 16 * i + 1 for i in range(8)]
    lay = Layout(sizes)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    srcs = [lay.random(bb, seed=100 + i) for i in range(slots)]
    host = [lay.objects(s.cpu().numpy()) for s in srcs]
    dsts = [lay.guarded() for _ in range(slots)]
    torch.cuda.synchronize()  # the side streams do not order after the current one

    def batch(i, algo, dst, verify_bad=None):
        want = [_model(bb, algo)(b) for b in host[i]]
        flags = bb.XFER_VERIFY if verify_bad is not None else 0
        items = [(srcs[i].data_ptr() + o, dst.data_ptr() + o, n, w ^ (k == verify_bad), flags)
                 for k, (o, n, w) in enumerate(zip(lay.offs, sizes, want))]
        return items, want

    order = ["CRC32C", "BBH64", "XXH3", "NONE"]
    tickets = []
    for i, algo in enumerate(order):
        items, want = batch(i, algo, dsts[i], verify_bad=2 if algo == "BBH64" else None)
        tickets.append((eng.submit(items, getattr(bb.ChecksumAlgo, algo), streams[i % 2].cuda_stream), want, algo))
    for i in reversed(range(slots)):
        t, want, algo = tickets[i]
        dg, st, _ = eng.wait(t)
        assert list(dg) == want, algo
        assert list(st) == [int(algo == "BBH64" and k == 2) for k in range(len(sizes))], algo
    torch.cuda.synchronize()
    for i in range(slots):
        lay.check(dsts[i], srcs[i], f"in-flight batch {i}")
    # submit i takes slot i when all are free: slot i runs cycle[(i + shift) % 3] in each round, and the shifts make every
    # slot see every ordered pair of the three algorithms
    cycle = ["BBH64", "XXH3", "CRC32C"]
    for rnd, shift in enumerate([0, 1, 2, 0, 2, 1, 0]):
        tickets = []
        for i in range(slots):
            algo = cycle[(i + shift) % 3]
            dsts[i].fill_(GUARD)
            items, want = batch(i, algo, dsts[i])
            tickets.append((eng.submit(items, getattr(bb.ChecksumAlgo, algo), _stream()), want, algo))
        for t, want, algo in tickets:
            dg, st, _ = eng.wait(t)
            assert list(dg) == want, (rnd, algo)
            assert list(st) == [0] * len(sizes)
        torch.cuda.synchronize()
        for i in range(slots):
            lay.check(dsts[i], srcs[i], f"round {rnd} batch {i}")


def test_raw_tensor_core_accumulators(bb, eng):
    """run(debug=True): the raw wgmma accumulators D[m][n] of every tile equal the integer product of the tile, laid out by
    bbh64_off_to_row / bbh64_off_to_k and zero padded, with the BBH64 weights (the model of _bbh64_numpy in
    test_common.py).  A full tile, a partial tail tile and the tile of a hash-only slice."""
    W = np.array([[bb.bbh64_weight(k, c) for c in range(16)] for k in range(128)], dtype=np.int64)
    o = np.arange(T)
    rows = np.array([bb.bbh64_off_to_row(int(v)) for v in o])
    ks = np.array([bb.bbh64_off_to_k(int(v)) for v in o])
    lay = Layout([T + 5000, 2000])
    src = lay.random(bb, seed=9)
    dst = lay.guarded()
    items = [(src.data_ptr(), dst.data_ptr(), T + 5000),
             (src.data_ptr() + lay.offs[1], [], 2000, 0, bb.XFER_RAW_SUM, 3)]
    eng.set_max_ctas(2)
    dg, _, _ = eng.run(items, bb.ChecksumAlgo.BBH64, _stream(), True)
    host = src.cpu().numpy()
    acc = np.array(eng.debug_accumulators(), dtype=np.uint32).reshape(3, 128, 16)
    tiles = [host[0:T], host[T:T + 5000], host[lay.offs[1]:lay.offs[1] + 2000]]
    for t, b in enumerate(tiles):
        tile = np.zeros(T, dtype=np.int64)
        tile[:len(b)] = b
        A = np.zeros((128, 128), dtype=np.int64)
        A[rows, ks] = tile
        D = A @ W
        assert np.array_equal(acc[t].astype(np.int64), D), f"tile {t}: rows {np.nonzero((acc[t] != D).any(axis=1))[0][:8]}"
    assert dg[0] == bb.bbh64(host[:T + 5000])
    assert dg[1] == bb.bbh64_partial(np.concatenate([np.zeros(3 * T, dtype=np.uint8), tiles[2]]), 3, 1)
