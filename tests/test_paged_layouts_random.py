"""Seeded random batches through XferEngine.run and run_fp8 that mix the three newest ways the fused kernels find their
bytes -- sparse page tables, in-page row patterns (XFER_PAGE_ROWS) and block ids resolved on the device -- with every
item kind of test_xfer_random.py, against host models; then the resolve kernel at its limits, and a regression test
for verdicts of mixed batches.

A byte round mixes test_xfer_random's items with sparse paged gets (a null first page, last page, one between stored
neighbours, or many), row-pattern puts (repeated pages) and gets (null pages), and blocks puts and gets: int32 and
int64 ids written on the caller's stream just before the call, 1 to 64 slices (a put's may alias), selections,
row patterns, tables rebased to a random byte (first > 0, phase != 0) and items that cover a prefix of what is left;
some ids are refused (out of range, negative, int64 >= 2^32, a get's duplicates and duplicate selection entries, a
duplicate pair at the first and last positions, duplicates together with an out-of-range id).  Some rounds are small or
mailbox rounds with one such item, which sends the batch to bb_xfer.  An fp8 round packs from row patterns and blocks
and unpacks into row patterns, blocks and sparse tables, in bf16, fp16 and fp32, sometimes reading as another type;
row widths in elements let 32-element MX blocks straddle rows and pages.

The models (test_paged_layouts_random_cpu.py): resolve() for block tables and verdicts, model_addr() for where each
byte lives; the digest models of test_common.py; the exact MXFP8 models of test_mxfp8_exhaustive.py and
test_mxfp8_wide.py.  Every destination byte and every guard byte is checked; a refused get stores nothing; every
non-BLOCKS item's verdict is OK.  Every failure names the seed, the round and the item.  BB_RANDOM_ROUNDS=k runs k more
rounds per seed."""
import collections

import numpy as np
import pytest
import torch

import test_xfer_random as xr
from test_paged_layouts_random_cpu import REFUSALS_GET, REFUSALS_PUT, Arena, blocks_table, page_table, placed, resolve

pytestmark = pytest.mark.gpu

T = 16384
MiB = 1 << 20
GUARD = 0xA5
ALGOS = ["NONE", "CRC32C", "BBH64", "XXH3"]
BYTE_SEEDS = [101, 211, 307, 401]
BYTE_ROUNDS = 30 + xr.EXTRA
FP8_SEEDS = [7, 17, 27]
FP8_ROUNDS = 12 + xr.EXTRA
NEW = ["spget", "rput", "rget", "bput", "bget"]
DUPS = ["dup", "dup-ends", "dup-sel"]  # drawn twice as often among a get's refusals: they are the ones only gets have
SEEN = collections.Counter()
DONE = set()


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need CUDA (marked gpu)")
    free, _ = torch.cuda.mem_get_info()
    if free < (5 << 29):
        pytest.skip(f"needs about 2.5 GiB of free device memory, {free >> 20} MiB free")


@pytest.fixture(scope="module")
def eng():
    from blackbird_b200 import _bb

    e = _bb.XferEngine(0, 4096, 2)
    yield e
    e.set_max_ctas(0)
    e.set_small_path(True)
    e.set_mailbox(True)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _codes(bb):
    return {0: bb.ErrorCode.OK, 1: bb.ErrorCode.VALUE_OUT_OF_RANGE, 2: bb.ErrorCode.INVALID_ARGUMENT}


class Ids:
    """Block ids (or selection entries) that the engine reads on the device: zeros until write() copies the real ones on
    the current stream, right before the call, with no host synchronize in between."""

    def __init__(self, a):
        self.real = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        self.dev = torch.zeros_like(self.real)

    def write(self):
        self.dev.copy_(self.real)


def device_blocks(bb, t, ptr, scale=1):
    """The DeviceBlocks of blocks_table() `t` whose cache lies at byte `ptr` + offset * scale, rebased to its offset."""
    t["_ids"] = Ids(t["ids"])
    t["_sel"] = None if t["sel"] is None else Ids(t["sel"])
    return bb.DeviceBlocks([ptr + int(o) * scale for o in t["outer"]], t["_ids"].dev.data_ptr(), t["ids"].size, t["n_blocks"],
                           t["stride"] * scale, t["page"], id_bytes=t["ids"].itemsize,
                           sel=0 if t["sel"] is None else t["_sel"].dev.data_ptr(), n_stored=t["n_stored"],
                           row_width=t["rw"], row_pitch=t["rp"]).rebase(t["off"])


def write_ids(ts):
    for t in ts:
        if "_ids" in t:
            t["_ids"].write()
            if t["_sel"] is not None:
                t["_sel"].write()


def where_bytes(t):
    """(object offsets, buffer offsets) of what an item over table `t` reads or stores, null pages left out."""
    if "outer" in t:
        return placed(t["table"][t["off"] // t["page"]:], t["page"], t["off"] % t["page"], t["rw"], t["rp"], t["n"])
    return placed(t["offs"], t["page"], t["phase"], t["rw"], t["rp"], t["n"])


# ---------------------------------------------------------------------------------------------------- byte items
class LItem(xr.Item):
    """A byte item whose gathered source or scattered destination is a sparse table, a row pattern or blocks."""

    def __init__(self, bb, rng, kind, sa, da, small, one_dst):
        super().__init__(kind, "")
        get = kind.endswith("get")
        budget = 1 << 14 if small else 1 << 21
        refuse = None
        if kind[0] == "b" and rng.random() < 0.35:
            refuse = str(rng.choice(REFUSALS_GET + DUPS if get else REFUSALS_PUT))
        arena = da if get else sa
        # half the blocks tables without a row pattern, so that every (pattern, selection, rebase) combination is common
        self.t = blocks_table(rng, arena, budget * 4, get, rows=rng.random() < 0.6, refuse=refuse) if kind[0] == "b" else \
            page_table(rng, arena, budget, get, rows=kind != "spget")
        self.verdict = self.t.get("verdict", 0)
        n = self.t["n"]
        xs, ds = where_bytes(self.t)
        if get:
            self.src = (sa.take(n), n)
            self.stores = [] if self.verdict else [(0, xs, ds)]
            self.dst_offs = [0]
        else:
            self.src = (None, n)
            self.src_at = ds
            self.dst_offs = [da.take(n) for _ in range(1 if one_dst else int(rng.integers(1, 4)))]
            self.stores = [(d, None, None) for d in self.dst_offs]
        self.desc = f"{kind} {self.t['what']} ndst={len(self.dst_offs)}"
        if rng.random() < 0.5:
            self.flags |= bb.XFER_VERIFY
            self.wrong = rng.random() < 0.5
            self.desc += " verify=" + ("wrong" if self.wrong else "right")

    @property
    def forced(self):
        return True

    def obj(self, host):
        if self.kind.endswith("get"):
            o, n = self.src
            return host[o:o + n]
        return host[self.src_at]

    def layout(self, bb, src_ptr, dst_ptr):
        t = self.t
        get = self.kind.endswith("get")
        ptr = dst_ptr if get else src_ptr
        if "outer" in t:
            return device_blocks(bb, t, ptr)
        return ([ptr + int(o) if o else 0 for o in t["offs"]], t["page"], t["phase"], t["rw"], t["rp"])

    def tuple(self, bb, src_ptr, dst_ptr, expect):
        lay = self.layout(bb, src_ptr, dst_ptr)
        n = self.t["n"]
        if self.kind.endswith("get"):
            slots = [None] * (4 if self.kind[0] != "b" else 6) + [lay]  # destination pages, or destination blocks
            return (src_ptr + self.src[0], [dst_ptr], n, expect, self.flags, 0, *slots)
        dsts = [dst_ptr + o for o in self.dst_offs]
        slots = [None] * (3 if self.kind[0] != "b" else 5) + [lay]  # source pages, or source blocks
        return (src_ptr, dsts, n, expect, self.flags, 0, *slots)


def _plan(rng, algo):
    """(mode, kinds): a mixed round of old and new kinds, or a small / mailbox round with one new-kind item."""
    if rng.random() < 0.3:
        mode = "mailbox" if rng.random() < 0.4 else "small"
        count = int(rng.integers(1, 9)) if mode == "mailbox" else int(rng.integers(1, 40))
        kinds = ["whole"] * count if mode == "mailbox" else [str(rng.choice(["whole", "zero", "verify-ok", "verify-bad"])) for _ in range(count)]
        kinds[int(rng.integers(0, count))] = str(rng.choice(NEW))
        return mode, kinds
    old = [k for k in xr.KINDS if algo in ("BBH64", "XXH3") or not k.startswith("slice")]
    count = int(rng.choice([int(rng.integers(1, 9)), int(rng.integers(9, 40))]))
    return "mixed", [str(rng.choice(NEW)) if rng.random() < 0.5 else str(rng.choice(old)) for _ in range(count)]


def byte_round(bb, eng, seed, rnd):
    rng = np.random.default_rng([seed, rnd, 1])
    algo = ALGOS[int(rng.integers(0, 4))]
    A = getattr(bb.ChecksumAlgo, algo)
    grid = xr._grid(rng)
    mode, kinds = _plan(rng, algo)
    sa, da = xr.Arena(rng), xr.Arena(rng)
    items = []
    for k in kinds:
        if k in NEW:
            items.append(LItem(bb, rng, k, sa, da, small=mode != "mixed", one_dst=mode == "mailbox"))
        else:
            items.append(xr.make_item(bb, rng, k, sa, da, small=mode != "mixed", one_dst=mode == "mailbox"))
    where = f"seed {seed} round {rnd} ({algo}, grid {grid}, {mode}, {len(items)} items)"
    src = torch.empty(sa.total, dtype=torch.uint8, device="cuda")
    dst = torch.empty(da.total, dtype=torch.uint8, device="cuda")
    fill_seed = seed * 1000 + rnd
    bb.random_fill(src.data_ptr(), src.numel(), fill_seed, _stream())
    host = src.cpu().numpy()
    digests = [it.digest(bb, algo, host) for it in items]
    tuples = []
    for it, d in zip(items, digests):
        expect = d ^ 1 if it.wrong else d
        tuples.append(it.tuple(bb, src.data_ptr(), dst.data_ptr(), expect) if isinstance(it, LItem) else
                      it.tuple(src.data_ptr(), dst.data_ptr(), expect))
    src.zero_()
    dst.fill_(GUARD)
    bb.random_fill(src.data_ptr(), src.numel(), fill_seed, _stream())
    write_ids([it.t for it in items if isinstance(it, LItem)])
    eng.set_max_ctas(grid)
    eng.set_mailbox(mode == "mailbox")
    if mode == "mailbox":
        torch.cuda.synchronize()
    blocks = any(isinstance(it, LItem) and it.kind[0] == "b" for it in items)
    before = (eng.launches, eng.small_launches, eng.mailbox_requests, eng.mailbox_launches)
    res = eng.run(tuples, A, _stream())
    torch.cuda.synchronize()
    dg, st = res[0], res[1]
    verdicts = res[3] if len(res) == 4 else [bb.ErrorCode.OK] * len(items)
    assert (len(res) == 4) == blocks, f"{where}: results {len(res)}"
    launches, small, mail, mail_launches = (a - b for a, b in zip((eng.launches, eng.small_launches, eng.mailbox_requests,
                                                                    eng.mailbox_launches), before))
    busy = [it for it in items if it.src and it.src[1] > 0 and not (algo == "NONE" and it.win is not None and it.win[1] <= it.win[0])]
    all_small = all(it.kind in ("whole", "verify-ok", "verify-bad") and it.src[1] <= 4096 for it in busy)
    if not busy:
        path, want = "none", (0, 0, 0)
    elif mode != "mixed" and any(it.forced for it in busy):
        path, want = "forced", (1, 0, 0)
    elif mode == "mailbox":
        path, want = "mailbox", (0, 0, len(busy))
    elif all_small:
        path, want = "warp", (1, 1, 0)
    else:
        path, want = "fused", (1, 0, 0)
    want = (want[0] + int(blocks), want[1], want[2])  # the resolve kernel is one launch more
    assert (launches - mail_launches, small, mail) == want, f"{where}: ran (launches, small, mailbox) = {(launches - mail_launches, small, mail)}, want the {path} path"
    if path == "forced":  # by what the forced items hold: blocks, or an in-page row pattern (XFER_PAGE_ROWS)
        lay = [it for it in items if isinstance(it, LItem)]
        SEEN[("forced", "blocks")] += any(it.kind[0] == "b" for it in lay)
        SEEN[("forced", "rows")] += any(it.kind[0] != "b" and it.t["rw"] != 0 for it in lay)
    SEEN[path] += 1
    codes = _codes(bb)
    for i, (it, d, s, v) in enumerate(zip(items, dg, st, verdicts)):
        want_d = 0 if algo == "NONE" else digests[i]
        want_s = int(algo != "NONE" and bool(it.flags & bb.XFER_VERIFY) and it.wrong)
        want_v = codes[it.verdict] if isinstance(it, LItem) else bb.ErrorCode.OK
        assert (d, s, v) == (want_d, want_s, want_v), \
            f"{where}, item {i} [{it.desc}]: digest {d:#x} status {s} verdict {v}, want {want_d:#x} status {want_s} verdict {want_v}"
        SEEN[(it.kind, algo)] += 1
        if isinstance(it, LItem):
            SEEN[("verdict", it.kind, it.verdict)] += 1
            if it.kind[0] == "b":
                t = it.t
                SEEN[("blocks", "rows" if t["rw"] else "plain", "sel" if t["sel"] is not None else "all",
                      "rebased" if t["off"] else "whole")] += 1
    want = np.full(dst.numel(), GUARD, dtype=np.uint8)
    owner = np.full(dst.numel(), -1, dtype=np.int32)
    for i, it in enumerate(items):
        b = it.obj(host)
        for base, xs, ds in it.stores:
            if xs is None:
                want[base:base + b.size] = b
                owner[base:base + b.size] = i
            elif xs.size:
                want[base + ds] = b[xs]
                owner[base + ds] = i
    got = dst.cpu().numpy()
    bad = np.nonzero(got != want)[0]
    if bad.size:
        first = int(bad[0])
        near = owner[max(0, first - 64):first + 64]
        idx = sorted({int(v) for v in near if v >= 0})
        pytest.fail(f"{where}: {bad.size} destination bytes differ, first at {first} (got {got[first]:#x}, want {want[first]:#x}); "
                    f"items near it: {[(i, items[i].desc) for i in idx]}")


@pytest.mark.parametrize("seed", BYTE_SEEDS)
def test_random_layout_byte_batches(bb, eng, seed):
    """Random batches mixing every byte kind with sparse, row-pattern and blocks items: bytes, guards, digests, status,
    verdicts and path."""
    for rnd in range(BYTE_ROUNDS):
        byte_round(bb, eng, seed, rnd)
    DONE.add(("bytes", seed))


# ---------------------------------------------------------------------------------------------------- MXFP8 items
MX_PACK = ["rows", "blocks"]
MX_UNPACK = ["rows", "blocks", "sparse"]
NPT = {2: np.uint16, 4: np.uint32}


def _mx_table(rng, arena, form, get, per, n_budget):
    """A table in elements for an fp8 item, its element count a positive multiple of 32 (None: draw again)."""
    for _ in range(20):
        refuse = None
        if form == "blocks" and rng.random() < 0.4:
            refuse = str(rng.choice(REFUSALS_GET + DUPS if get else REFUSALS_PUT))
        t = blocks_table(rng, arena, n_budget, get, per=per, refuse=refuse) if form == "blocks" else \
            page_table(rng, arena, n_budget, get, per=per, rows=form == "rows")
        n = t["n"] // 32 * 32
        if n == 0:
            continue
        t["n"] = n
        return t
    return None


def fp8_round(bb, eng, seed, rnd):
    rng = np.random.default_rng([seed, rnd, 8])
    mx = {"bf16": bb.MxWide.BF16, "f16": bb.MxWide.F16, "f32": bb.MxWide.F32}
    codes = _codes(bb)
    eng.set_max_ctas(xr._grid(rng))
    side = xr.SIDES[int(rng.random() < 0.4)]
    where = f"fp8 seed {seed} round {rnd} ({side})"

    def types(s, k):
        return ["f32" if s == "fp32" else str(rng.choice(["bf16", "f16"])) for _ in range(k)]

    # ---- pack from row patterns and blocks
    count = int(rng.integers(1, 7))
    ws = types(side, count)
    b = xr.WB[ws[0]]
    per = 16 // b
    ar = Arena(rng)
    forms = [str(rng.choice(MX_PACK)) for _ in range(count)]
    tabs = []
    for f in forms:
        t = None
        while t is None:
            t = _mx_table(rng, ar, f, False, per, 1 << 18)
        tabs.append(t)
    host = np.full(ar.total, xr.WGUARD[b], dtype=NPT[b])
    for t, w in zip(tabs, ws):  # values where each item reads (for a refused put, block 0 of every slice)
        _, ds = where_bytes(t)
        host[ds] = xr._values(rng, w, -(-ds.size // 32) * 32)[:ds.size]
    dev = torch.from_numpy(host.view(np.int16 if b == 2 else np.int32).copy()).cuda()
    objs = [host[where_bytes(t)[1]] for t in tabs]
    packed = [xr._pack_model(x, w) for x, w in zip(objs, ws)]
    lay = xr.Layout([p.size for p in packed])
    out = lay.guarded()
    items = []
    for t, w, o in zip(tabs, ws, lay.offs):
        n = t["n"]
        if "outer" in t:
            lay_ = device_blocks(bb, t, dev.data_ptr(), scale=b)
            items.append((0, [out.data_ptr() + o], n, None, None, None, None, mx[w], None, None, lay_))
        else:
            pg = ([dev.data_ptr() + b * int(v) for v in t["offs"]], t["page"], t["phase"], t["rw"], t["rp"])
            items.append((0, [out.data_ptr() + o], n, None, None, None, None, mx[w], pg))
    descs = [f"{w} {f} {t['what']} (n={t['n']} after rounding to MX blocks)" for w, f, t in zip(ws, forms, tabs)]
    write_ids(tabs)
    res = eng.run_fp8(items, False, _stream(), wide=mx[ws[0]])
    torch.cuda.current_stream().synchronize()
    blocks = any("outer" in t for t in tabs)
    assert (len(res) == 4) == blocks, where
    verdicts = res[3] if blocks else [bb.ErrorCode.OK] * count
    got = out.cpu().numpy()
    for i, (t, p) in enumerate(zip(tabs, packed)):
        v = t.get("verdict", 0)
        assert verdicts[i] == codes[v] and res[1][i] == 0, f"{where}, item {i} [{descs[i]}]: verdict {verdicts[i]}"
        assert res[0][i] == bb.bbh64(p), f"{where}, item {i} [{descs[i]}]: digest"
        o = lay.offs[i]
        xr.same_bits(got[o:o + t["n"]], p[:t["n"]], "e4m3", f"{where}, item {i} [{descs[i]}]: payload")
        xr.same_bits(got[o + t["n"]:o + p.size], p[t["n"]:], "e8m0", f"{where}, item {i} [{descs[i]}]: scales")
        SEEN[("pack", ws[i], forms[i])] += 1
        SEEN[("verdict", "fp8-pack", v)] += 1
    outside = np.ones(lay.total, dtype=bool)
    for o, p in zip(lay.offs, packed):
        outside[o:o + p.size] = False
    assert bool((got[outside] == GUARD).all()), f"{where}: pack wrote outside its objects"
    # ---- unpack into row patterns, blocks and sparse tables, sometimes as a type of the other size
    gside = side if rng.random() < 0.7 else xr.SIDES[1 - xr.SIDES.index(side)]
    count = int(rng.integers(1, 7))
    gws = types(gside, count)
    pws = types(side, count)  # the type each object was packed from
    gb = xr.WB[gws[0]]
    gper = 16 // gb
    ar = Arena(rng)
    uforms = [str(rng.choice(MX_UNPACK)) for _ in range(count)]
    utabs = []
    for f in uforms:
        t = None
        while t is None:
            t = _mx_table(rng, ar, f, True, gper, 1 << 18)
        utabs.append(t)
    upacked = [xr._pack_model(xr._values(rng, w, t["n"]), w) for t, w in zip(utabs, pws)]
    ulay = xr.Layout([p.size for p in upacked])
    pbuf = np.full(ulay.total, GUARD, dtype=np.uint8)
    for o, p in zip(ulay.offs, upacked):
        pbuf[o:o + p.size] = p
    pdev = torch.from_numpy(pbuf).cuda()
    odev = torch.full((ar.total,), xr.WGUARD[gb], dtype=torch.int16 if gb == 2 else torch.int32, device="cuda")
    wrong = [bool(rng.random() < 0.25) for _ in range(count)]
    gets = []
    for i, (t, w, o, p) in enumerate(zip(utabs, gws, ulay.offs, upacked)):
        expect = bb.bbh64(p) ^ int(wrong[i])
        if "outer" in t:
            gets.append((0, pdev.data_ptr() + o, t["n"], expect, None, None, None, mx[w], None, None, None,
                         device_blocks(bb, t, odev.data_ptr(), scale=gb)))
        else:
            pg = ([odev.data_ptr() + gb * int(v) if v else 0 for v in t["offs"]], t["page"], t["phase"], t["rw"], t["rp"])
            gets.append((0, pdev.data_ptr() + o, t["n"], expect, None, None, None, mx[w], None, pg))
    udescs = [f"packed from {pw}, get as {w} {f} {t['what']} (n={t['n']} after rounding to MX blocks)" for pw, w, f, t in zip(pws, gws, uforms, utabs)]
    write_ids(utabs)
    res = eng.run_fp8(gets, True, _stream(), wide=mx[gws[0]])
    torch.cuda.current_stream().synchronize()
    blocks = any("outer" in t for t in utabs)
    verdicts = res[3] if blocks else [bb.ErrorCode.OK] * count
    got = odev.cpu().numpy().view(NPT[gb])
    want = np.full(ar.total, xr.WGUARD[gb], dtype=NPT[gb])
    for i, (t, p) in enumerate(zip(utabs, upacked)):
        v = t.get("verdict", 0)
        assert (verdicts[i], res[1][i]) == (codes[v], int(wrong[i])), f"{where}, item {i} [{udescs[i]}]: verdict {verdicts[i]} status {res[1][i]}"
        if not v:
            xs, ds = where_bytes(t)
            want[ds] = xr._unpack_model(p, t["n"], gws[i])[xs]
        SEEN[("unpack", gws[i], uforms[i])] += 1
        SEEN[("verdict", "fp8-unpack", v)] += 1
        SEEN[("cross", gside)] += gws[i] != pws[i]
    written = np.zeros(ar.total, dtype=bool)
    for i, (t, w) in enumerate(zip(utabs, gws)):  # each item in its own type: a NaN only has to be a NaN of that type
        xs, ds = where_bytes(t)
        if ds.size and not t.get("verdict", 0):
            written[ds] = True
            xr._same(got[ds], want[ds], w, f"{where}, item {i} [{udescs[i]}]: unpacked")
    outside = np.nonzero(~written & (got != xr.WGUARD[gb]))[0]
    assert outside.size == 0, f"{where}: unpack wrote {outside.size} elements outside its results, first at {outside[:4].tolist()}"


@pytest.mark.parametrize("seed", FP8_SEEDS)
def test_random_layout_fp8_batches(bb, eng, seed):
    """Random MXFP8 packs from row patterns and blocks and unpacks into row patterns, blocks and sparse tables, against
    the exact models."""
    for rnd in range(FP8_ROUNDS):
        fp8_round(bb, eng, seed, rnd)
    DONE.add(("fp8", seed))


def test_every_layout_kind_verdict_and_forced_path_occurred():
    """The rounds above reached every new kind x algorithm, every verdict of blocks puts and gets, and the forced
    bb_xfer path of a small or mailbox round with a rows item and with a blocks item, at least 3 times each."""
    if len(DONE) < len(BYTE_SEEDS) + len(FP8_SEEDS):
        pytest.skip("runs only after every random test of this module ran")
    missing = [(k, a, SEEN[(k, a)]) for k in NEW for a in ALGOS if SEEN[(k, a)] < 3]
    missing += [(k, v, SEEN[("verdict", k, v)]) for k, vs in (("bput", (0, 1)), ("bget", (0, 1, 2))) for v in vs
                if SEEN[("verdict", k, v)] < 3]
    missing += [("forced", f, SEEN[("forced", f)]) for f in ("rows", "blocks") if SEEN[("forced", f)] < 3]
    missing += [(op, w, f, SEEN[(op, w, f)]) for w in xr.WIDES for op, forms in (("pack", MX_PACK), ("unpack", MX_UNPACK))
                for f in forms if SEEN[(op, w, f)] < 3]
    missing += [("fp8 verdict", op, v, SEEN[("verdict", op, v)]) for op, vs in (("fp8-pack", (0, 1)), ("fp8-unpack", (0, 1, 2)))
                for v in vs if SEEN[("verdict", op, v)] < 3]
    missing += [("blocks", r, s, b, SEEN[("blocks", r, s, b)]) for r in ("rows", "plain") for s in ("sel", "all")
                for b in ("rebased", "whole") if SEEN[("blocks", r, s, b)] < 3]
    print("\ncoverage:", {str(k): v for k, v in sorted(SEEN.items(), key=str)})
    assert not missing, f"categories reached too rarely: {missing}"


# ---------------------------------------------------------------------------------------------------- deterministic
def _rand(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=g)


def _blocks(bb, keep, cache_ptr, ids, n_blocks, stride, page, dtype=torch.int32, sel=None, n_stored=0):
    """DeviceBlocks over one slice at cache_ptr; the id tensors are kept alive in `keep`."""
    i = torch.tensor(ids, dtype=dtype, device="cuda")
    s = None if sel is None else torch.tensor(sel, dtype=dtype, device="cuda")
    keep += [i, s]
    return bb.DeviceBlocks([cache_ptr], i.data_ptr(), len(ids), n_blocks, stride, page, id_bytes=i.element_size(),
                           sel=0 if s is None else s.data_ptr(), n_stored=n_stored)


def _get(src_ptr, n, blocks, expect=0, flags=0):
    return (src_ptr, 0, n, expect, flags, 0, None, None, None, None, None, None, blocks)


def test_a_mixed_batch_after_a_refused_blocks_get_reports_ok_verdicts(bb):
    """A refused blocks get leaves its verdict at its descriptor's index of the slot; the next batch of that slot puts a
    contiguous item, a paged get and a row-pattern get there, with a good blocks get behind them: every verdict is OK,
    in XferEngine.run and in run_fp8."""
    E, A = bb.ErrorCode, bb.ChecksumAlgo.XXH3
    eng = bb.XferEngine(0, 64, 1)  # one slot: every run below takes it
    keep = []
    page = 4096
    src = _rand(8 * page, 1)
    cache = torch.full((16 * page,), GUARD, dtype=torch.uint8, device="cuda")
    res = eng.run([_get(src.data_ptr(), 2 * page, _blocks(bb, keep, cache.data_ptr(), [3, 3], 16, page, page)),
                   _get(src.data_ptr(), 2 * page, _blocks(bb, keep, cache.data_ptr(), [1, 16], 16, page, page)),
                   _get(src.data_ptr(), 2 * page, _blocks(bb, keep, cache.data_ptr(), [2, 4], 16, page, page, sel=[0, 0], n_stored=2))],
                  A, _stream())
    torch.cuda.synchronize()
    assert res[3] == [E.INVALID_ARGUMENT, E.VALUE_OUT_OF_RANGE, E.INVALID_ARGUMENT] and bool((cache == GUARD).all())
    out = torch.zeros(2 * page, dtype=torch.uint8, device="cuda")
    pages = torch.full((4 * page,), GUARD, dtype=torch.uint8, device="cuda")
    rows = torch.full((8 * page,), GUARD, dtype=torch.uint8, device="cuda")
    p0, r0 = pages.data_ptr(), rows.data_ptr()
    res = eng.run([(src.data_ptr(), out.data_ptr(), 2 * page),
                   (src.data_ptr(), 0, 2 * page, 0, 0, 0, None, None, None, None, ([p0 + 2 * page, 0, p0], page, 0)),
                   (src.data_ptr(), 0, 2 * page, 0, 0, 0, None, None, None, None, ([r0 + 4 * page, r0], page, 0, 1024, 2048)),
                   _get(src.data_ptr(), 2 * page, _blocks(bb, keep, cache.data_ptr(), [5, 9], 16, page, page))], A, _stream())
    torch.cuda.synchronize()
    assert res[3] == [E.OK] * 4 and res[1] == [0] * 4
    assert torch.equal(out, src[:2 * page]) and torch.equal(cache[5 * page:6 * page], src[:page]) and torch.equal(cache[9 * page:10 * page], src[page:2 * page])
    assert torch.equal(pages[2 * page:3 * page], src[:page]) and bool((pages[:2 * page] == GUARD).all()) and bool((pages[3 * page:] == GUARD).all())
    assert torch.equal(rows.view(-1, 1024)[[16, 18, 20, 22, 0, 2, 4, 6]].reshape(-1), src[:2 * page])
    # run_fp8: unpack into blocks refused, then a plain unpack in front of a good blocks unpack
    n = 2 * 2048  # bf16 elements: two pages of 2048
    wide = torch.randn(n, device="cuda").to(torch.bfloat16)
    packed = torch.full((n + n // 32,), GUARD, dtype=torch.uint8, device="cuda")
    dg, _, _ = eng.run_fp8([(wide.data_ptr(), [packed.data_ptr()], n)], False, _stream())
    cache.fill_(GUARD)
    res = eng.run_fp8([(0, packed.data_ptr(), n, dg[0], None, None, None, None, None, None, None,
                        _blocks(bb, keep, cache.data_ptr(), [7, 7], 16, page, 2048))], True, _stream())
    torch.cuda.synchronize()
    assert res[3] == [E.INVALID_ARGUMENT] and bool((cache == GUARD).all())
    back = torch.zeros_like(wide)
    res = eng.run_fp8([(back.data_ptr(), packed.data_ptr(), n, dg[0]),
                       (0, packed.data_ptr(), n, dg[0], None, None, None, None, None, None, None,
                        _blocks(bb, keep, cache.data_ptr(), [2, 11], 16, page, 2048))], True, _stream())
    torch.cuda.synchronize()
    assert res[3] == [E.OK, E.OK] and res[1] == [0, 0]
    assert torch.equal(cache[2 * page:3 * page], back.view(torch.uint8)[:page]) and torch.equal(cache[11 * page:12 * page], back.view(torch.uint8)[page:])


M = 1 << 18  # kBlocksMaxDistinct: bits of the resolve kernel's duplicate bitmap


def test_resolve_kernel_at_the_distinct_bound(bb, eng):
    """n_blocks and n_stored of 2^18 resolve for a get; 2^18 + 1 is NOT_IMPLEMENTED before any launch; a put with
    2^18 + 1 blocks resolves and reads block 2^18.  The selection pass at that bound with first > 0 and a partial count
    (a rebased table) stores exactly the selected pages it covers."""
    E, A = bb.ErrorCode, bb.ChecksumAlgo.XXH3
    keep = []
    cache = torch.full(((M + 1) * 16,), GUARD, dtype=torch.uint8, device="cuda")
    obj = _rand(M * 16, 2)
    ids = [M - 1, 0, 12345, M // 2]
    dg, st, _, v = eng.run([_get(obj.data_ptr(), 64, _blocks(bb, keep, cache.data_ptr(), ids, M, 16, 16))], A, _stream())
    torch.cuda.synchronize()
    assert v == [E.OK] and st == [0]
    want = torch.full_like(cache, GUARD).view(-1, 16)
    want[torch.tensor(ids, device="cuda")] = obj[:64].view(-1, 16)
    assert torch.equal(cache, want.view(-1))
    for kw in (dict(n_blocks=M + 1), dict(n_blocks=8, sel=[M, 1, 2, 3], n_stored=M + 1)):
        b = _blocks(bb, keep, cache.data_ptr(), [1, 2, 3, 4], kw["n_blocks"], 16, 16, sel=kw.get("sel"), n_stored=kw.get("n_stored", 0))
        before = eng.launches
        with pytest.raises(RuntimeError, match="NOT_IMPLEMENTED"):
            eng.run([_get(obj.data_ptr(), b.npages * 16, b)], A, _stream())
        assert eng.launches == before
    torch.cuda.synchronize()
    assert torch.equal(cache, want.view(-1))
    # a put may name more blocks than the bitmap covers
    out = torch.zeros(48, dtype=torch.uint8, device="cuda")
    _, _, _, v = eng.run([(0, out.data_ptr(), 48, 0, 0, 0, None, None, None, None, None,
                           _blocks(bb, keep, cache.data_ptr(), [M, 0, M - 1], M + 1, 16, 16, dtype=torch.int64))], A, _stream())
    torch.cuda.synchronize()
    assert v == [E.OK] and torch.equal(out.view(-1, 16), cache.view(-1, 16)[[M, 0, M - 1]])
    # n_stored == 2^18: an object of 2^18 pages, three of them stored; then the same table rebased past page 2^18 - 5
    for off, n in ((0, M * 16), ((M - 5) * 16 + 7, 5 * 16 - 7), ((M - 5) * 16 + 7, 3 * 16)):
        at = (16 - off % 16) % 16  # the slice's address + phase 16-byte aligned
        buf = torch.full((8 * 16 + 32,), GUARD, dtype=torch.uint8, device="cuda")
        small = buf[at:at + 8 * 16]
        sel = [M - 1, 0, M - 3]
        b = _blocks(bb, keep, small.data_ptr(), [5, 1, 7], 8, 16, 16, dtype=torch.int64, sel=sel, n_stored=M).rebase(off)
        part = obj[off:off + n].clone()  # a get's contiguous source starts 16-byte aligned
        _, st, _, v = eng.run([_get(part.data_ptr(), n, b)], A, _stream())
        torch.cuda.synchronize()
        assert v == [E.OK] and st == [0], off
        assert bool((buf[:at] == GUARD).all()) and bool((buf[at + 8 * 16:] == GUARD).all()), off
        w = torch.full_like(small, GUARD).view(-1, 16)
        for blk, s in zip([5, 1, 7], sel):
            lo, hi = max(s * 16, off), min((s + 1) * 16, off + n)
            if lo < hi:
                w[blk, lo - s * 16:hi - s * 16] = obj[lo:hi]
        assert torch.equal(small, w.view(-1)), (off, n)


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
def test_resolve_kernel_with_100k_ids(bb, eng, dtype):
    """100,000 distinct ids, far more than the kernel's 512 threads: a permutation resolves for a put and a get; the same
    with a duplicate pair at the first and last positions is refused and stores nothing."""
    E, A = bb.ErrorCode, bb.ChecksumAlgo.CRC32C
    keep = []
    K, NB = 100_000, 100_017
    perm = np.random.default_rng(5).permutation(NB)[:K]
    cache = _rand(NB * 16, 3)
    out = torch.zeros(K * 16, dtype=torch.uint8, device="cuda")
    _, _, _, v = eng.run([(0, out.data_ptr(), K * 16, 0, 0, 0, None, None, None, None, None,
                           _blocks(bb, keep, cache.data_ptr(), perm.tolist(), NB, 16, 16, dtype=dtype))], A, _stream())
    torch.cuda.synchronize()
    idx = torch.from_numpy(perm).cuda()
    assert v == [E.OK] and torch.equal(out.view(-1, 16), cache.view(-1, 16)[idx])
    dst = torch.full_like(cache, GUARD)
    obj = _rand(K * 16, 4)
    _, st, _, v = eng.run([_get(obj.data_ptr(), K * 16, _blocks(bb, keep, dst.data_ptr(), perm.tolist(), NB, 16, 16, dtype=dtype))], A, _stream())
    torch.cuda.synchronize()
    want = torch.full_like(dst, GUARD).view(-1, 16)
    want[idx] = obj.view(-1, 16)
    assert v == [E.OK] and st == [0] and torch.equal(dst, want.view(-1))
    dup = perm.copy()
    dup[-1] = dup[0]
    dst.fill_(GUARD)
    _, _, _, v = eng.run([_get(obj.data_ptr(), K * 16, _blocks(bb, keep, dst.data_ptr(), dup.tolist(), NB, 16, 16, dtype=dtype))], A, _stream())
    torch.cuda.synchronize()
    assert v == [E.INVALID_ARGUMENT] and bool((dst == GUARD).all())


def test_hundreds_of_blocks_items_carry_their_own_verdicts(bb, eng):
    """One batch of 400 BLOCKS items, one resolve CTA each, puts and gets with refused ones scattered among them: each
    item reports its own verdict, refused gets store nothing, the others store exactly their blocks."""
    E, A = bb.ErrorCode, bb.ChecksumAlgo.BBH64
    codes = _codes(bb)
    rng = np.random.default_rng(9)
    keep, items, plan = [], [], []
    N, NB, P = 400, 12, 64
    cache = _rand(N * NB * P, 6)
    dst = torch.full((N * NB * P,), GUARD, dtype=torch.uint8, device="cuda")
    src = _rand(N * 4 * P, 7)
    out = torch.full((N * 4 * P,), GUARD, dtype=torch.uint8, device="cuda")
    for i in range(N):
        get = bool(i % 2)
        ids = rng.permutation(NB)[:4]
        kind = int(rng.integers(0, 5)) if rng.random() < 0.3 else 0
        if kind == 1:
            ids[int(rng.integers(0, 4))] = NB
        elif kind == 2:
            ids[int(rng.integers(0, 4))] = -2
        elif kind >= 3:
            ids[3] = ids[0]  # a get's duplicate, a put's repeat
        verdict, table = resolve([0], ids, NB, P, get=get)
        base = i * NB * P
        if get:
            items.append(_get(src.data_ptr() + i * 4 * P, 4 * P, _blocks(bb, keep, dst.data_ptr() + base, ids.tolist(), NB, P, P)))
        else:
            items.append((0, out.data_ptr() + i * 4 * P, 4 * P, 0, 0, 0, None, None, None, None, None,
                          _blocks(bb, keep, cache.data_ptr() + base, ids.tolist(), NB, P, P, dtype=torch.int64)))
        plan.append((get, verdict, table + base))
    _, st, _, v = eng.run(items, A, _stream())
    torch.cuda.synchronize()
    assert v == [codes[p[1]] for p in plan] and st == [0] * N
    assert {p[1] for p in plan if p[0]} == {0, 1, 2} and {p[1] for p in plan if not p[0]} == {0, 1}
    c, s = cache.cpu().numpy(), src.cpu().numpy()
    want_dst = np.full(dst.numel(), GUARD, dtype=np.uint8)
    want_out = np.full(out.numel(), GUARD, dtype=np.uint8)
    for i, (get, verdict, table) in enumerate(plan):
        for k, a in enumerate(table):
            if get and not verdict:
                want_dst[a:a + P] = s[i * 4 * P + k * P:i * 4 * P + (k + 1) * P]
            elif not get:
                want_out[i * 4 * P + k * P:i * 4 * P + (k + 1) * P] = c[a:a + P]
    assert np.array_equal(dst.cpu().numpy(), want_dst) and np.array_equal(out.cpu().numpy(), want_out)
