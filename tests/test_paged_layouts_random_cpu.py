"""Seeded random paged layouts on CPU: sparse page tables, in-page row patterns and block ids, drawn by the generators
that test_paged_layouts_random.py also drives through XferEngine on the GPU, against independent numpy models.

The models here are the ones the GPU rounds trust:
  - resolve(): the SourceBlocks rule written out with explicit loops (verdict order: out of range before duplicate; a
    refused get's table all null, a refused put's block 0 of each slice), checked against model_table / model_verdict of
    test_layer_blocks_cpu.py and against DeviceBlocks.resolve at random rebases;
  - model_addr() of test_paged_rows_cpu.py for where object byte x lives in a table with an in-page row pattern.
Then random sequences of the paged and blocks client calls through the HostLoopbackTransport, with 1-3 replicas and
1-2 workers per copy, so that shards start mid-page and mid-row: the loopback runs SourceBlocks::resolve and
for_each_run at every shard cut, and every byte of every cache, guards included, is compared with the model.
Every failure names the seed, the step and the item.  BB_RANDOM_ROUNDS=k runs k more steps per seed."""
import math
import os

import numpy as np
import pytest

from blackbird_b200.parallel import LocalCluster
from test_layer_blocks_cpu import model_table, model_verdict
from test_paged_rows_cpu import model_addr

T = 16384
GUARD = 0xA5
MiB = 1 << 20
EXTRA = int(os.environ.get("BB_RANDOM_ROUNDS", "0"))


# ---------------------------------------------------------------------------------------------------- models
def resolve(outer, ids, n_blocks, stride, sel=None, n_stored=0, get=False):
    """(verdict 0 OK / 1 out of range / 2 duplicate, every page entry of the object) by the SourceBlocks rule."""
    ids = [int(v) for v in ids]
    sel = None if sel is None else [int(v) for v in sel]
    out = any(v < 0 or v >= n_blocks for v in ids) or (sel is not None and any(s < 0 or s >= n_stored for s in sel))
    dup = get and (len(set(ids)) != len(ids) or (sel is not None and len(set(sel)) != len(sel)))
    verdict = 1 if out else 2 if dup else 0
    per = len(ids) if sel is None else n_stored
    table = np.zeros(len(outer) * per, dtype=np.int64)
    for q, o in enumerate(outer):
        if verdict:
            table[q * per:(q + 1) * per] = 0 if get else o
            continue
        for m, b in enumerate(ids):
            table[q * per + (m if sel is None else sel[m])] = o + b * stride
    return verdict, table


def placed(table, page, phase, rw, rp, n):
    """(object offsets, addresses) of the object bytes [0, n) that land: those in a non-null page of the table."""
    x = np.arange(n, dtype=np.int64)
    t = np.asarray(table, dtype=np.int64)
    live = t[(x + phase) // page] != 0
    return x[live], model_addr(t, page, phase, rw, rp, x[live])


# ---------------------------------------------------------------------------------------------------- generators
def row_pattern(rng, per=16, tile=T, rows=True):
    """(page, row_width, row_pitch, what) in units of which `per` make 16 bytes: in-page rows of one granule (a tile then
    holds 1024 of them), of a width that is no multiple of a granule (only the gap is), or wider than a tile; or no
    pattern.  The page is a multiple of a granule."""
    kind = str(rng.choice(["granule", "odd", "wide"])) if rows and rng.random() < 0.8 else "none"
    if kind == "none":
        page = per * int(rng.choice([1, 3, 2 * int(rng.integers(0, 300)) + 1, tile // per, tile // per + 1, 4 * int(rng.integers(1, 40))]))
        return page, 0, 0, f"page={page}"
    if kind == "granule":
        rw, nrows = per, int(rng.choice([2, 3, int(rng.integers(2, 1100))]))
    else:
        rw = int(rng.integers(1, 12 * per)) if kind == "odd" else tile + int(rng.integers(1, 3 * per))
        if rw % per == 0:
            rw += 1
        unit = per // math.gcd(rw, per)  # at least 2: rows of this many make a page of whole granules
        nrows = unit * int(rng.integers(1, 4 if kind == "odd" else 2))
    rp = rw + per * int(rng.choice([1, 2, int(rng.integers(1, 24))]))
    return rw * nrows, rw, rp, f"page={rw * nrows} rows {rw}/{rp} ({kind})"


def extent(page, rw, rp):
    """Units from a page's address to the end of its last row."""
    return page if rw == 0 else (page // rw - 1) * rp + rw


def _phase(rng, page):
    return int(rng.choice([0, int(rng.integers(0, page)), page - 1]))


def page_table(rng, arena, budget, get, per=16, rows=True, phase_ok=True):
    """A page table for a put (repeated pages) or a get (null pages: none, the first, the last, one between stored
    neighbours or many, never all): dict(offs (0 = null), page, phase, rw, rp, n, what).  Regions lie in `arena`
    (units), page k's address + phase a multiple of 16 bytes."""
    page, rw, rp, what = row_pattern(rng, per, rows=rows)
    npages = max(1, min(int(rng.choice([1, 2, int(rng.integers(1, 40)), int(rng.integers(40, 1500))])), budget // page))
    phase = _phase(rng, page) if phase_ok else 0
    lo = max(1, (npages - 1) * page - phase + 1)
    hi = npages * page - phase
    n = hi if not phase_ok else int(rng.choice([lo, hi, int(rng.integers(lo, hi + 1))]))
    offs = arena.pages(npages, extent(page, rw, rp), residue=(-phase) % per, mod=per)
    offs = offs[rng.permutation(npages)]
    note = ""
    if not get and npages > 1 and rng.random() < 0.25:
        k = rng.integers(0, npages, max(1, npages // 4))
        offs[k] = offs[rng.integers(0, npages, k.size)]
        note = f" repeats={k.size}"
    if get and npages > 1 and rng.random() < 0.7:
        mode = str(rng.choice(["first", "last", "inner", "many"]))
        if mode == "first":
            offs[0] = 0
        elif mode == "last":
            offs[-1] = 0
        elif mode == "inner" and npages > 2:
            offs[int(rng.integers(1, npages - 1))] = 0
        else:
            k = rng.permutation(npages)[:int(rng.integers(1, npages))]
            offs[k] = 0
        note = f" nulls={int((offs == 0).sum())} ({mode})"
    return dict(offs=offs, page=page, phase=phase, rw=rw, rp=rp, n=n, what=f"{what} phase={phase} pages={npages}{note} n={n}")


REFUSALS_PUT = ["high", "neg", "huge"]
REFUSALS_GET = ["high", "neg", "huge", "sel-high", "dup", "dup-ends", "dup-sel", "dup+high"]


def blocks_table(rng, arena, budget, get, per=16, rows=True, phase_ok=True, refuse=None):
    """Blocks of a cache in `arena`: 1 to 64 slices (a put's may alias), ids of 4 or 8 bytes, for a get sometimes a
    selection; `refuse` breaks one rule (REFUSALS_*); with phase_ok the table is rebased to a random unit (first > 0,
    phase != 0) and the item covers a random prefix of what is left.  dict(outer, ids, sel, n_stored, n_blocks,
    stride, page, rw, rp, off, n, verdict, table (every page), what)."""
    page, rw, rp, what = row_pattern(rng, per, rows=rows)
    ext = extent(page, rw, rp)
    stride = -(-ext // per) * per + per * int(rng.choice([0, 0, 1, 3]))
    n_outer = int(rng.choice([1, 2, int(rng.integers(1, 9)), int(rng.integers(9, 65))]))
    n_ids = int(rng.choice([1, 2, int(rng.integers(1, 12)), int(rng.integers(12, 100))]))
    n_blocks = n_ids + int(rng.choice([0, int(rng.integers(0, 16))]))
    while n_outer > 1 and n_outer * n_blocks * stride > budget:
        n_outer //= 2
    while n_ids > 1 and n_outer * n_blocks * stride > budget:
        n_ids //= 2
        n_blocks = n_ids + (n_blocks - n_ids) // 2
    if refuse in ("dup", "dup-ends", "dup-sel", "dup+high") and n_ids < 2:
        n_ids, n_blocks = 2, max(n_blocks, 2)
    dt = np.int32 if rng.random() < 0.5 else np.int64
    ids = rng.permutation(n_blocks)[:n_ids].astype(np.int64)
    if not get and n_ids > 1 and rng.random() < 0.3:  # a put may repeat ids
        ids = rng.integers(0, n_blocks, n_ids).astype(np.int64)
    sel, n_stored = None, 0
    if get and (rng.random() < 0.4 or refuse in ("sel-high", "dup-sel")):
        n_stored = n_ids + int(rng.choice([0, int(rng.integers(0, 6))]))
        sel = rng.permutation(n_stored)[:n_ids].astype(np.int64)
    if refuse == "huge":
        dt = np.int64
    k = int(rng.integers(0, n_ids))
    if refuse == "high":
        ids[k] = n_blocks + int(rng.choice([0, int(rng.integers(0, 1000))]))
    elif refuse == "neg":
        ids[k] = -1 - int(rng.choice([0, int(rng.integers(0, 1 << 30))]))
    elif refuse == "huge":
        ids[k] = (1 << 32) + int(rng.choice([0, int(ids[k])]))  # its low 32 bits are a valid id
    elif refuse == "sel-high":
        sel[k] = n_stored
    elif refuse == "dup":
        a, b = rng.permutation(n_ids)[:2]
        ids[b] = ids[a]
    elif refuse == "dup-ends":
        ids[-1] = ids[0]
    elif refuse == "dup-sel":
        sel[-1] = sel[0]
    elif refuse == "dup+high":  # both broken: out of range comes first
        ids[-1] = ids[0]
        ids[k] = n_blocks
    ids = ids.astype(dt)
    if sel is not None:
        sel = sel.astype(dt)
    per_outer = n_ids if sel is None else n_stored
    total = n_outer * per_outer * page
    off = int(rng.choice([0, int(rng.integers(0, total)), (int(rng.integers(0, n_outer * per_outer))) * page + page - 1])) if phase_ok and rng.random() < 0.5 else 0
    phase = off % page
    step = n_blocks * stride if get else stride * int(rng.integers(1, n_blocks + 1))  # a put's slices may alias
    base = arena.take((n_outer - 1) * step + n_blocks * stride, residue=(-phase) % per, mod=per)
    outer = [base + q * step for q in range(n_outer)]
    left = total - off
    n = left if not phase_ok or rng.random() < 0.5 else int(rng.integers(1, left + 1))
    v, table = resolve(outer, ids, n_blocks, stride, sel, n_stored, get)
    what = (f"{what} slices={n_outer} ids={n_ids}x{np.dtype(dt).itemsize}B blocks={n_blocks} stride={stride}"
            f"{'' if sel is None else f' sel of {n_stored}'} off={off} n={n}{'' if refuse is None else f' refused={refuse}'}")
    return dict(outer=outer, ids=ids, sel=sel, n_stored=n_stored, n_blocks=n_blocks, stride=stride, page=page, rw=rw, rp=rp,
                off=off, n=n, verdict=v, table=table, what=what)


class Arena:
    """Regions of a buffer of units, each at a chosen residue mod `mod`, with guard units between them (as
    test_xfer_random.Arena, whose page method this shares)."""

    def __init__(self, rng):
        self.rng, self.end = rng, 16

    def take(self, n, residue=0, mod=16):
        o = self.end + mod + int(self.rng.integers(0, 2 * mod))
        o += (residue - o) % mod
        self.end = o + n
        return o

    def pages(self, count, n, residue=0, mod=16):
        step = (n + mod - 1) // mod * mod
        gaps = mod * self.rng.integers(1, 4, count)
        start = self.end + mod + (residue - self.end - mod) % mod
        offs = start + np.arange(count, dtype=np.int64) * step + np.cumsum(gaps) - gaps[0]
        self.end = int(offs[-1]) + n
        return offs

    @property
    def total(self):
        return self.end + 64


# ---------------------------------------------------------------------------------------------------- the models checked
def test_resolve_matches_the_layer_blocks_model_and_device_blocks(bb):
    """resolve() agrees with model_table / model_verdict and, at random rebases, with DeviceBlocks.resolve, the reference
    the loopback runs; refusals of every kind come out in the documented order."""
    E = bb.ErrorCode
    codes = {0: E.OK, 1: E.VALUE_OUT_OF_RANGE, 2: E.INVALID_ARGUMENT}
    rng = np.random.default_rng(71)
    seen = set()
    for trial in range(400):
        get = bool(trial % 2)
        refuse = None if rng.random() < 0.5 else str(rng.choice(REFUSALS_GET if get else REFUSALS_PUT))
        t = blocks_table(rng, Arena(rng), 1 << 20, get, refuse=refuse)
        ids = t["ids"].astype(np.int64)
        sel = None if t["sel"] is None else t["sel"].astype(np.int64)
        mv = model_verdict(ids, t["n_blocks"], sel, t["n_stored"], get)
        assert t["verdict"] == mv, (trial, t["what"])
        assert np.array_equal(t["table"], model_table(t["outer"], ids, t["stride"], sel, t["n_stored"], mv, get)), (trial, t["what"])
        seen.add((get, t["verdict"]))
        b = bb.DeviceBlocks([int(o) + (1 << 32) for o in t["outer"]], t["ids"].ctypes.data, t["ids"].size, t["n_blocks"], t["stride"],
                            t["page"], id_bytes=t["ids"].itemsize, sel=0 if t["sel"] is None else t["sel"].ctypes.data,
                            n_stored=t["n_stored"], row_width=t["rw"], row_pitch=t["rp"]).rebase(t["off"])
        r0 = t["off"] // t["page"]
        count = (t["n"] - 1 + t["off"] % t["page"]) // t["page"] + 1
        assert (b.first, b.phase) == (r0, t["off"] % t["page"]) and b.valid(t["n"]), t["what"]
        v, table = b.resolve(count, get)
        want = t["table"][r0:r0 + count]
        want = np.where(want != 0, want + (1 << 32), 0)
        assert v == codes[t["verdict"]] and np.array_equal(np.asarray(table, dtype=np.int64), want), (trial, t["what"])
    assert seen == {(False, 0), (False, 1), (True, 0), (True, 1), (True, 2)}


def test_generated_tables_follow_the_engine_rules(bb):
    """Every table the generators draw is one the engine takes: valid and co-aligned, a put's without a null page; and
    SourcePages.runs over it visits exactly the bytes placed() names."""
    rng = np.random.default_rng(72)
    for trial in range(300):
        get = bool(trial % 2)
        ar = Arena(rng)
        t = page_table(rng, ar, 1 << 20, get)
        base = 1 << 32
        addrs = [base + int(o) if o else 0 for o in t["offs"]]
        xs, ds = placed(t["offs"], t["page"], t["phase"], t["rw"], t["rp"], t["n"])
        if not get:
            assert xs.size == t["n"], t["what"]
        ec, p, _ = bb.SourcePages.from_pages(addrs, t["page"], t["rw"], t["rp"])
        assert ec == bb.ErrorCode.OK, t["what"]
        r = p.rebase(t["phase"])
        assert r.coaligned(t["n"]) and r.phase == t["phase"], t["what"]
        got_x, got_a = [], []
        for x, at, m in r.runs(t["n"]):
            got_x.append(np.arange(x, x + m))
            got_a.append(np.arange(at, at + m, dtype=np.int64))
        gx = np.concatenate(got_x) if got_x else np.zeros(0, np.int64)
        ga = np.concatenate(got_a) if got_a else np.zeros(0, np.int64)
        assert np.array_equal(gx, xs) and np.array_equal(ga - base, ds), (trial, t["what"])
        # the regions hold what they are read or stored at, and no two pages of a get overlap
        live = ds.size and get
        if live:
            assert np.unique(ds).size == ds.size, t["what"]
        assert ar.total > int(ds.max(initial=0)), t["what"]


# ---------------------------------------------------------------------------------------------------- loopback sequences
def make_client(bb, c):
    cl = c.client(node_id="node-0")
    io = c.client(node_id="node-0")
    bb.attach_loopback_transport(cl, io, False)
    return cl


class Host:
    """A guard-filled host buffer addressed in units from a 16-byte aligned base."""

    def __init__(self, units):
        self.raw = np.full(units + 64, GUARD, dtype=np.uint8)
        self.o0 = (-self.raw.ctypes.data) % 16
        self.buf = self.raw[self.o0:self.o0 + units]

    def addr(self, o):
        return self.buf.ctypes.data + int(o) if o else 0


def _blocks(bb, h, t):
    return bb.DeviceBlocks([h.addr(o) for o in t["outer"]], t["ids"].ctypes.data, t["ids"].size, t["n_blocks"], t["stride"], t["page"],
                           id_bytes=t["ids"].itemsize, sel=0 if t["sel"] is None else t["sel"].ctypes.data, n_stored=t["n_stored"],
                           row_width=t["rw"], row_pitch=t["rp"])


def loopback_step(bb, cl, seed, step, seen):
    """Puts from random row-pattern tables and blocks (some refused), each read back whole; gets of stored objects into
    sparse tables, row patterns and blocks (some refused); every cache byte against the model."""
    E = bb.ErrorCode
    codes = {0: E.OK, 1: E.VALUE_OUT_OF_RANGE, 2: E.INVALID_ARGUMENT}
    rng = np.random.default_rng([seed, step])
    replicas, stripes = int(rng.integers(1, 4)), int(rng.integers(1, 3))
    cfg = bb.WorkerConfig(replication_factor=replicas, max_workers_per_copy=stripes, ttl_ms=0,
                          checksum=bb.ChecksumAlgo.XXH3 if rng.random() < 0.7 else bb.ChecksumAlgo.NONE,
                          preferred_classes=[bb.StorageClass.RAM_CPU])
    where = f"seed {seed} step {step} (replicas {replicas}, workers {stripes})"
    ar = Arena(rng)
    kinds = [str(rng.choice(["rput", "bput", "spget", "rget", "bget"])) for _ in range(int(rng.integers(1, 5)))]
    items = []
    for k in kinds:
        get = k.endswith("get")
        refuse = None
        if k.startswith("b") and rng.random() < 0.25:
            refuse = str(rng.choice(REFUSALS_GET if get else REFUSALS_PUT))
        if k.startswith("b"):
            items.append((k, blocks_table(rng, ar, 1 << 20, get, phase_ok=False, refuse=refuse)))
        else:
            items.append((k, page_table(rng, ar, 1 << 19, get, rows=k != "spget", phase_ok=False)))
    h = Host(ar.total)
    h.buf[:] = np.frombuffer(os.urandom(h.buf.size), dtype=np.uint8)
    src = h.buf.copy()  # what the puts read: the caches before any get writes them
    want = h.buf.copy()
    for i, (k, t) in enumerate(items):
        key = f"{seed}/{step}/{i}"
        desc = f"{where}, item {i} [{k} {t['what']}]"
        if k.endswith("put"):
            if k == "rput":
                ecs = cl.batch_put_device_paged([key], [[h.addr(o) for o in t["offs"]]], [t["page"]], cfg, 0,
                                                rows=[(t["rw"], t["rp"]) if t["rw"] else None])
                v, table = 0, t["offs"]
            else:
                ecs = cl.batch_put_device_blocks([key], [_blocks(bb, h, t)], cfg, 0)
                v, table = t["verdict"], t["table"]
            assert ecs == [codes[v]], f"{desc}: {ecs}"
            seen[(k, "verdict", v)] += 1
            if v:
                assert not cl.object_exists(key), desc
                continue
            n = len(table) * t["page"]
            xs, ds = placed(table, t["page"], 0, t["rw"], t["rp"], n)
            assert np.array_equal(np.frombuffer(cl.get(key), dtype=np.uint8), src[ds]), desc
        else:
            n = (len(t["table"]) if k == "bget" else len(t["offs"])) * t["page"]
            obj = np.frombuffer(os.urandom(n), dtype=np.uint8)
            assert cl.put(key, obj.tobytes(), cfg) == E.OK, desc
            if k == "bget":
                ecs, sizes = cl.batch_get_device_blocks([key], [_blocks(bb, h, t)], 0)
                v, table = t["verdict"], t["table"]
            else:
                ecs, sizes = cl.batch_get_device_paged([key], [[h.addr(o) for o in t["offs"]]], [t["page"]], 0,
                                                       rows=[(t["rw"], t["rp"]) if t["rw"] else None])
                v, table = 0, t["offs"]
            assert ecs == [codes[v]], f"{desc}: {ecs}"
            seen[(k, "verdict", v)] += 1
            if not v:
                xs, ds = placed(table, t["page"], 0, t["rw"], t["rp"], n)
                want[ds] = obj[xs]
        got = h.buf
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, f"{desc}: {bad.size} bytes differ, first at {bad[0]}"
        seen[k] += 1


@pytest.mark.parametrize("seed", [3, 19])
def test_random_loopback_sequences(bb, seed):
    import collections

    seen = collections.Counter()
    with LocalCluster(cluster_id=f"plr{seed}", n_workers=4, pool_bytes=256 * MiB) as c:
        cl = make_client(bb, c)
        for step in range(12 + EXTRA):
            loopback_step(bb, cl, seed, step, seen)
    assert all(seen[k] >= 1 for k in ("rput", "bput", "spget", "rget", "bget")), dict(seen)
