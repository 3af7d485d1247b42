"""Launch geometry of the fused transfer kernel: short CTAs of at most 8 tiles, two resident per SM, for NONE, XXH3 and
BBH64, one persistent CTA per SM for CRC32C.  Runs that start and end mid-object are combined by the finalizers' cross-CTA
path, so every check here compares the bytes, digests and verify status of a launch at the default geometry with the
CPU models and with a launch of one CTA per SM (set_max_ctas), bit for bit."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

T = 16384
GUARD = 0xA5
ALGOS = ["NONE", "CRC32C", "BBH64", "XXH3"]
RUN = 8  # tiles per CTA run of the default geometry (kRunTiles)


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


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _model(bb, algo):
    return {"NONE": lambda b: 0, "CRC32C": bb.crc32c, "BBH64": bb.bbh64, "XXH3": bb.xxh3t64}[algo]


def _random(bb, n, seed):
    t = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
    bb.random_fill(t.data_ptr(), t.numel(), seed, _stream())
    return t


def _cdiv(a, b):
    return (a + b - 1) // b


def expected_grid(algo, tiles, sms):
    """cta_tile_run gives each CTA ceil(tiles / grid) tiles; CTAs that would get none are not launched."""
    grid = sms if algo == "CRC32C" else max(min(2 * sms, tiles), _cdiv(tiles, RUN))
    grid = min(grid, tiles)
    return _cdiv(tiles, _cdiv(tiles, grid))


@pytest.mark.parametrize("algo", ALGOS)
def test_default_geometry(bb, algo):
    """Stages, residency and grid: two 6-stage CTAs per SM (the occupancy query agrees) except for CRC32C's one 8-stage
    CTA; at most one tile per CTA up to twice the SM count, at most RUN (8) tiles per CTA for large batches."""
    A = getattr(bb.ChecksumAlgo, algo)
    sms = _sms()
    g = bb.xfer_geometry(A, 1)
    crc = algo == "CRC32C"
    assert (g["stages"], g["resident_ctas_per_sm"]) == ((8, 1) if crc else (6, 2)), g
    assert g["resident_ctas_per_sm"] * (g["smem_bytes"] + 1024) <= 228 * 1024
    for tiles in (1, 5, sms, 2 * sms, 2 * sms + 1, 300, 64 * sms + 1, 12360, 262144):
        got = bb.xfer_geometry(A, tiles)["grid"]
        assert got == expected_grid(algo, tiles, sms), (tiles, got)
        if not crc:
            assert _cdiv(tiles, got) <= (1 if tiles <= 2 * sms else RUN), (tiles, got)
    # an explicit grid still wins
    assert bb.xfer_geometry(A, 262144, 7)["grid"] == 7
    assert bb.xfer_geometry(A, 1000, 2 * sms)["grid"] == _cdiv(1000, _cdiv(1000, 2 * sms))


@pytest.mark.parametrize("algo", ALGOS)
def test_whole_objects_match_models_and_one_cta_per_sm(bb, eng, algo):
    """Objects of 1, 33 and 4096 tiles, each also with a partial tile, a sub-tile object and a second 4096-tile object
    (12360 tiles: more than 8 per CTA at twice the SM count), 1-3 destinations each, verified: the default geometry and a
    grid of one CTA per SM give the same bytes, digests and status, and the digests equal the CPU models."""
    A = getattr(bb.ChecksumAlgo, algo)
    sizes = [T, 33 * T, 4096 * T, T + 5, 33 * T + 100, 4096 * T + 1, 100, 4096 * T]
    assert sum(_cdiv(n, T) for n in sizes) == 12360
    offs = np.cumsum([0] + [_cdiv(n, 64) * 64 for n in sizes])
    src = _random(bb, int(offs[-1]), 5)
    host = src.cpu().numpy()
    model = _model(bb, algo)
    digests = [model(host[o:o + n]) for o, n in zip(offs, sizes)]
    ndst = [1 + i % 3 for i in range(len(sizes))]
    regions, o = [], 64
    for n, k in zip(sizes, ndst):
        rs = []
        for _ in range(k):
            rs.append(o)
            o = _cdiv(o + n + 64, 16) * 16
        regions.append(rs)
    dst = torch.full((o + 64,), GUARD, dtype=torch.uint8, device="cuda")
    flags = bb.XFER_VERIFY if algo != "NONE" else 0
    items = [(src.data_ptr() + int(so), [dst.data_ptr() + r for r in rs], n, d, flags) for so, n, rs, d in zip(offs, sizes, regions, digests)]
    want = np.full(dst.numel(), GUARD, dtype=np.uint8)
    for so, n, rs in zip(offs, sizes, regions):
        for r in rs:
            want[r:r + n] = host[so:so + n]
    results = []
    for g in (0, _sms()):
        eng.set_max_ctas(g)
        dst.fill_(GUARD)
        dg, st, _ = eng.run(items, A, _stream())
        torch.cuda.synchronize()
        assert st == [0] * len(sizes), (g, st)
        assert np.array_equal(dst.cpu().numpy(), want), g
        results.append((dg, st))
    assert results[0] == results[1]
    if algo != "NONE":
        assert results[0][0] == digests
        # a wrong expected digest is reported by the object's status only
        bad = list(items)
        bad[5] = bad[5][:3] + (digests[5] ^ 1, flags)
        eng.set_max_ctas(0)
        _, st, _ = eng.run(bad, A, _stream())
        assert st == [0] * 5 + [1] + [0] * 2, st


@pytest.mark.parametrize("algo", ALGOS)
def test_windows_strides_and_gathers(bb, eng, algo):
    """One batch of ~12000 tiles holding a windowed get, a strided get, a gathered put and a plain item with three
    destinations, every object ~3000 tiles so that CTA runs start and end inside windows, rows and gathered rows: the same
    bytes, digests and status at the default geometry and at one CTA per SM, digests equal to the CPU models, and the tile
    trace keeps its four stamps per tile."""
    A = getattr(bb.ChecksumAlgo, algo)
    model = _model(bb, algo)
    n = 3000 * T + 77
    obj = _random(bb, n, 9)
    ohost = obj.cpu().numpy()
    pitch, width = 4016, 4000  # (pitch - width) % 16 == 0: rows co-aligned with the tile
    rows = _cdiv(n, width)
    gsrc = _random(bb, rows * pitch, 10)
    ghost = gsrc.cpu().numpy()
    gidx = np.arange(n, dtype=np.int64)
    dense = ghost[gidx // width * pitch + gidx % width]
    lo, hi = T - 3, 2000 * T + 5
    s = lo % 16  # the window's bytes start at win_buf + s, so object byte 0 would sit at a 16-byte aligned address
    win_buf = torch.full((hi - lo + 64,), GUARD, dtype=torch.uint8, device="cuda")
    str_buf = torch.full((n + 64,), GUARD, dtype=torch.uint8, device="cuda")
    gat_buf = torch.full((n + 64,), GUARD, dtype=torch.uint8, device="cuda")
    plain = [torch.full((n + 64,), GUARD, dtype=torch.uint8, device="cuda") for _ in range(3)]
    d_obj, d_dense = model(ohost.tobytes()), model(dense.tobytes())
    vf = bb.XFER_VERIFY if algo != "NONE" else 0
    items = [(obj.data_ptr(), win_buf.data_ptr() + s - lo, n, d_obj, vf, 0, (lo, hi)),
             (obj.data_ptr(), str_buf.data_ptr(), n, d_obj, vf, 0, (0, n, pitch, width, 0)),
             (gsrc.data_ptr(), gat_buf.data_ptr(), n, 0, 0, 0, None, (pitch, width, 0)),
             (obj.data_ptr(), [b.data_ptr() for b in plain], n, d_obj, vf)]
    x = np.arange(n, dtype=np.int64)
    keep = x % pitch < width
    want_str = np.full(str_buf.numel(), GUARD, dtype=np.uint8)
    want_str[(x // pitch * width + x % pitch)[keep]] = ohost[keep]
    want_win = np.full(win_buf.numel(), GUARD, dtype=np.uint8)
    want_win[s:s + hi - lo] = ohost[lo:hi]
    want_full = np.full(n + 64, GUARD, dtype=np.uint8)
    want_full[:n] = ohost
    want_gat = want_full.copy()
    want_gat[:n] = dense
    tiles = 4 * _cdiv(n, T)
    results = []
    for g in (0, _sms()):
        eng.set_max_ctas(g)
        for b in [win_buf, str_buf, gat_buf] + plain:
            b.fill_(GUARD)
        eng.set_tile_trace(g == 0)
        dg, st, _ = eng.run(items, A, _stream())
        torch.cuda.synchronize()
        if g == 0:
            tr = np.asarray(eng.tile_trace(), dtype=np.uint64).reshape(-1, 4).astype(np.int64)
            eng.set_tile_trace(False)
            # without a digest a windowed item loads only the tiles its window touches
            assert (tr.shape[0] == tiles if algo != "NONE" else 0 < tr.shape[0] < tiles) and (tr > 0).all(), tr.shape
            assert (tr[:, 2] >= tr[:, 1]).all() and (tr[:, 3] >= tr[:, 2]).all()
        assert st == [0] * 4, (g, st)
        assert np.array_equal(win_buf.cpu().numpy(), want_win), g
        assert np.array_equal(str_buf.cpu().numpy(), want_str), g
        assert np.array_equal(gat_buf.cpu().numpy(), want_gat), g
        for b in plain:
            assert np.array_equal(b.cpu().numpy(), want_full), g
        results.append((dg, st))
    assert results[0] == results[1]
    if algo != "NONE":
        assert results[0][0] == [d_obj, d_obj, d_dense, d_obj]
