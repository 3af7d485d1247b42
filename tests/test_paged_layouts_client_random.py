"""Seeded random operation sequences of the client's row-pattern and blocks calls on a GpuRankCluster (an HBM slab and a
DRAM pool the fused kernels reach over PCIe), against the host model of test_device_model_random.py.

LayoutModel adds to that model's store and checks: byte puts and gets through batch_put_device_paged /
batch_get_device_paged with rows= (row patterns from test_paged_layouts_random_cpu.row_pattern, null pages on gets,
some pages 8 bytes off alignment), batch_put_device_blocks / batch_get_device_blocks (whole and partial restores,
int32 and int64 ids written on the stream just before the call, refused ids, tables 8 bytes off alignment), and the
fp8 forms of all four, in bf16, fp16 and fp32 (objects sometimes read as another type).  Puts use 1-3 replicas and 1-2
workers per copy, so shards start mid-page and mid-row and the client rebases the tables at every cut
(SourceBlocks::rebase with first > 0 and phase != 0).

Each item's code is predicted from the rules in blackbird_client.h: a refused put is VALUE_OUT_OF_RANGE and cancelled
while the rest of the batch is stored; a blocks table that is not co-aligned is NOT_IMPLEMENTED (no host-staged path);
byte row and page tables that are not co-aligned on some shard are staged (counted by the client); a refused get stores
nothing; an fp8 get is NOT_IMPLEMENTED unless some copy is one shard on the fabric and its table is fused-aligned.  After
every step every copy's stored bytes and digest are checked (check_all), and every cache byte, guards included.
BB_RANDOM_ROUNDS=k runs 10k more steps per seed."""
import math
import os

import numpy as np
import pytest
import torch

import test_device_model_random as dm
from test_paged_layouts_random import device_blocks, write_ids
from test_paged_layouts_random_cpu import REFUSALS_GET, REFUSALS_PUT, Arena, blocks_table, extent, placed, resolve, row_pattern
from test_xfer_random import WB, WGUARD, WIDES, _pack_model, _same

pytestmark = pytest.mark.gpu

GUARD = 0xA5
SEEDS = [5, 23]
STEPS = 80 + int(os.environ.get("BB_RANDOM_ROUNDS", "0")) * 10
OPS = ["put_rows", "get_rows", "put_blocks", "get_blocks", "put_fp8_rows", "get_fp8_rows", "put_fp8_blocks", "get_fp8_blocks", "remove"]


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need CUDA (marked gpu)")
    free, _ = torch.cuda.mem_get_info()
    if free < (5 << 29):
        pytest.skip(f"needs about 2.5 GiB of free device memory, {free >> 20} MiB free")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def table_ok(addrs, page, rw, rp, off, length, get):
    """SourcePages::coaligned of the table rebased to object unit `off` over `length` units, in bytes (addresses, page and
    pattern already in bytes); get: fused_get_aligned, which also wants page % 16 for any table of several pages."""
    if get and len(addrs) > 1 and page % 16:
        return False
    ph, k0 = off % page, off // page
    n = (length - 1 + ph) // page + 1 if length else 0
    if (n > 1 and page % 16) or (n and rw and (rp - rw) % 16):
        return False
    return all(a == 0 or (a + ph) % 16 == 0 for a in addrs[k0:k0 + n])


def _divisors(n, per, limit):
    return [d for d in range(per, min(n, limit) + 1, per) if n % d == 0] or [n]


def rows_for(rng, n, per):
    """(page, row_width, row_pitch) in units for an object of n units that the pages hold exactly: the page divides n,
    a pattern's width divides the page and may be no multiple of 32 elements or 16 bytes."""
    page = int(rng.choice(_divisors(n, per, 1 << 15)))
    nrows = [r for r in (2, 3, 4, 5, 8, 16) if page % r == 0 and page // r > 0]
    if not nrows or rng.random() < 0.2:
        return page, 0, 0
    rw = page // int(rng.choice(nrows))
    return page, rw, rw + per * int(rng.choice([1, 2, int(rng.integers(1, 24))]))


class LayoutModel(dm.Model):
    def __init__(self, bb, cl, seed):
        super().__init__(bb, cl, seed)
        self.blocks = {}  # key -> (page, row_width, slices, ids) of a put from blocks, in units of the object

    def _cfg(self, fp8):
        algo = "BBH64" if fp8 else dm.ALGOS[int(self.rng.integers(0, 4))]
        reps, workers = int(self.rng.integers(1, 4)), int(self.rng.integers(1, 3))
        return dm._cfg(self.bb, algo, reps, str(self.rng.choice(["RAM_GPU", "RAM_CPU"])), workers), algo, reps, workers

    def _check_cache(self, got, want, items):
        bad = np.nonzero(got != want)[0]
        if bad.size:
            first = int(bad[0])
            pytest.fail(f"{self.where()}: {bad.size} wrong cache units, first at {first} (got {got[first]:#x}, want {want[first]:#x}); items {items}")

    def _outcome(self, i, desc, got, exp):
        assert got == exp, f"{self.where(i, desc)}: {got}, want {exp}"
        self.outcomes[str(exp).split(".")[-1]] += 1

    # ------------------------------------------------------------------------------------------------ row patterns
    def put_rows(self, fp8=False):
        bb, rng, E = self.bb, self.rng, self.bb.ErrorCode
        count = int(rng.integers(1, 5))
        w = str(rng.choice(WIDES)) if fp8 else None
        b = WB[w] if fp8 else 1
        per = 16 // b
        cfg, algo, reps, workers = self._cfg(fp8)
        ar = Arena(rng)
        specs = []
        for _ in range(count):
            page, rw, rp, what = row_pattern(rng, per)
            npg = int(rng.choice([1, 2, int(rng.integers(1, 40)), int(rng.integers(40, 400))]))
            npg = max(1, min(npg, (150000 // b) // page))
            if fp8:
                npg = -(-npg // (32 // math.gcd(page, 32))) * (32 // math.gcd(page, 32))  # whole MX blocks
            offs = ar.pages(npg, extent(page, rw, rp), mod=per)[rng.permutation(npg)]
            if npg > 1 and rng.random() < 0.25:
                k = rng.integers(0, npg, max(1, npg // 4))
                offs[k] = offs[rng.integers(0, npg, k.size)]
            skew = rng.random() < 0.2
            if skew:
                offs[int(rng.integers(0, npg))] += 1 if fp8 else 8
            specs.append((page, rw, rp, offs, f"{what} pages={npg} skew={skew}"))
        host = np.full(ar.total + 16, GUARD if not fp8 else WGUARD[b], dtype=np.uint8 if not fp8 else np.dtype(f"u{b}"))
        xs = []
        for page, rw, rp, offs, _ in specs:
            _, ds = placed(offs, page, 0, rw, rp, len(offs) * page)
            v = dm._wide(rng, -(-ds.size // 32) * 32, w)[:ds.size] if fp8 else rng.integers(0, 256, ds.size, dtype=np.uint8)
            host[ds] = v
            xs.append(host[ds].copy())  # a repeated page holds what was written last
        src = torch.from_numpy(host.view(np.uint8).copy()).cuda()
        p = src.data_ptr()
        keys = [self.new_key() for _ in specs]
        lists = [[p + b * int(o) for o in s[3]] for s in specs]
        rows = [(s[1], s[2]) if s[1] else None for s in specs]
        self.what = f"{'fp8 ' + w + ' ' if fp8 else ''}rows put of {count}, {algo}, {reps} replicas, {workers} workers per copy"
        st0 = self.counter("device_put_host_staged_total")
        if fp8:
            ecs = self.cl.client.batch_put_device_fp8_paged(keys, lists, [s[0] for s in specs], cfg, _stream(), wide=dm._mx(bb, w), rows=rows)
        else:
            ecs = self.cl.client.batch_put_device_paged(keys, lists, [s[0] for s in specs], cfg, _stream(), rows=rows)
        torch.cuda.synchronize()
        staged = 0
        for i, (k, (page, rw, rp, offs, desc), addrs, x) in enumerate(zip(keys, specs, lists, xs)):
            aligned = table_ok(addrs, page * b, rw * b, rp * b, 0, len(offs) * page * b, False)
            exp = E.NOT_IMPLEMENTED if fp8 and not aligned else E.OK
            self._outcome(i, f"{k} {desc}", ecs[i], exp)
            if exp != E.OK:
                continue
            self.objs[k] = dm.Obj(_pack_model(x, w), "BBH64", reps, None, x, w) if fp8 else dm.Obj(x, algo, reps, None)
            if not fp8:  # staged unless every shard of every copy is co-aligned
                staged += not all(table_ok(addrs, page, rw, rp, off, sh.length, False)
                                  for shs in self.shards(k) for off, sh in zip(dm._starts(shs), shs))
        assert self.counter("device_put_host_staged_total") - st0 == staged, f"{self.where()}: staged items"
        self.outcomes["rows put staged"] += staged

    def get_rows(self, fp8=False):
        bb, rng, E = self.bb, self.rng, self.bb.ErrorCode
        keys = self.pick(fp8, int(rng.integers(1, 5)), gone=0.2)
        if not keys:
            return
        gw = str(rng.choice(WIDES)) if fp8 else None
        gb = WB[gw] if fp8 else 1
        per = 16 // gb
        ar = Arena(rng)
        specs = []
        for k in keys:
            o = self.objs.get(k)
            n = (o.x.size if fp8 else o.data.size) if o else 32
            if fp8:
                page, rw, rp = rows_for(rng, n, per)
                npg = n // page
            else:
                page, rw, rp, _ = row_pattern(rng, per)
                while -(-n // page) > 4000:
                    page, rw, rp, _ = row_pattern(rng, per)
                npg = -(-n // page) + int(rng.choice([0, 0, 1]))  # a shorter object fills its pages in order
            offs = ar.pages(npg, extent(page, rw, rp), mod=per)[rng.permutation(npg)]
            if npg > 1 and rng.random() < 0.5:
                offs[rng.permutation(npg)[:int(rng.integers(1, npg))]] = 0  # null pages: a partial restore
            skew = rng.random() < 0.15
            if skew:  # a stored page off alignment (a null page stays null)
                live = np.nonzero(offs)[0]
                offs[int(rng.choice(live))] += 1 if fp8 else 8
            specs.append((k, o, n, page, rw, rp, offs))
        out = torch.full((ar.total + 16,), WGUARD[gb] if fp8 else GUARD, dtype={1: torch.uint8, 2: torch.int16, 4: torch.int32}[gb], device="cuda")
        p = out.data_ptr()
        lists = [[p + gb * int(a) if a else 0 for a in s[6]] for s in specs]
        rows = [(s[4], s[5]) if s[4] else None for s in specs]
        self.what = f"{'fp8 as ' + gw + ' ' if fp8 else ''}rows get of {len(keys)}"
        st0 = self.counter("device_get_host_staged_total")
        if fp8:
            ecs = self.cl.client.batch_get_device_fp8_paged(keys, lists, [s[3] for s in specs], _stream(), wide=dm._mx(bb, gw), rows=rows)
        else:
            ecs, sizes = self.cl.client.batch_get_device_paged(keys, lists, [s[3] for s in specs], _stream(), rows=rows)
        torch.cuda.synchronize()
        got = out.cpu().numpy().view({1: np.uint8, 2: np.uint16, 4: np.uint32}[gb])
        want = np.full(got.size, WGUARD[gb] if fp8 else GUARD, dtype=got.dtype)
        staged, items = 0, []
        for i, ((k, o, n, page, rw, rp, offs), addrs) in enumerate(zip(specs, lists)):
            desc = f"{k} n={n} page={page} rows {rw}/{rp} pages={len(offs)} nulls={int((offs == 0).sum())}"
            xs, ds = placed(offs, page, 0, rw, rp, n)

            def fused(off, ln):
                return table_ok(addrs, page * gb, rw * gb, rp * gb, off * gb, ln * gb, True)

            if o is None:
                exp = E.OBJECT_NOT_FOUND
            elif fp8:
                exp = E.OK if self._fp8_usable(k) and fused(0, n) else E.NOT_IMPLEMENTED
                if exp == E.OK:
                    want[ds] = o.back(gw)[xs]
                    _same(got[ds], want[ds], gw, self.where(i, desc))
                    got[ds] = want[ds]  # NaN patterns compared above; the guard check below is exact
                    self.outcomes["cross-type read"] += gw != o.w
            else:
                exp = E.OK
                assert sizes[i] == n, f"{self.where(i, desc)}: size {sizes[i]}"
                want[ds] = o.data[xs]
                staged += self.get_staged(k, fused)
            self._outcome(i, desc, ecs[i], exp)
            items.append(desc)
        self._check_cache(got, want, items)
        assert self.counter("device_get_host_staged_total") - st0 == staged, f"{self.where()}: staged items"
        self.outcomes["rows get staged"] += staged

    def put_fp8_rows(self):
        self.put_rows(fp8=True)

    def get_fp8_rows(self):
        self.get_rows(fp8=True)

    # ------------------------------------------------------------------------------------------------ blocks
    def put_blocks(self, fp8=False):
        bb, rng, E = self.bb, self.rng, self.bb.ErrorCode
        codes = {0: E.OK, 1: E.VALUE_OUT_OF_RANGE}
        count = int(rng.integers(1, 5))
        w = str(rng.choice(WIDES)) if fp8 else None
        b = WB[w] if fp8 else 1
        per = 16 // b
        cfg, algo, reps, workers = self._cfg(fp8)
        ar = Arena(rng)
        ts = []
        for _ in range(count):
            skew = rng.random() < 0.15
            refuse = None if skew or rng.random() < 0.75 else str(rng.choice(REFUSALS_PUT))
            # an object of whole MX blocks, or of a multiple of 32 bytes: shard cuts (size / workers) stay 16-byte aligned,
            # so that co-alignment is the table's alone
            t = None
            while t is None or (t["n"] * b) % 32 or (fp8 and t["n"] % 32):
                t = blocks_table(rng, ar, (1 << 20) // b, False, per=per, phase_ok=False, refuse=refuse)
            t["skew"] = skew
            ts.append(t)
        host = np.full(ar.total + 16, GUARD if not fp8 else WGUARD[b], dtype=np.uint8 if not fp8 else np.dtype(f"u{b}"))
        for t in ts:  # values in every page the table or its refusal reads
            _, ds = placed(t["table"], t["page"], 0, t["rw"], t["rp"], t["n"])
            host[ds] = dm._wide(rng, -(-ds.size // 32) * 32, w)[:ds.size] if fp8 else rng.integers(0, 256, ds.size, dtype=np.uint8)
        src = torch.from_numpy(host.view(np.uint8).copy()).cuda()
        keys = [self.new_key() for _ in ts]
        blocks = [device_blocks(bb, t, src.data_ptr() + (8 if t["skew"] else 0), scale=b) for t in ts]
        self.what = f"{'fp8 ' + w + ' ' if fp8 else ''}blocks put of {count}, {algo}, {reps} replicas, {workers} workers per copy"
        torch.cuda.synchronize()
        torch.cuda._sleep(20_000_000)  # the ids land behind a long kernel: the call must read them on the stream
        write_ids(ts)
        if fp8:
            ecs = self.cl.client.batch_put_device_fp8_blocks(keys, blocks, cfg, _stream(), wide=dm._mx(bb, w))
        else:
            ecs = self.cl.client.batch_put_device_blocks(keys, blocks, cfg, _stream())
        torch.cuda.synchronize()
        for i, (k, t) in enumerate(zip(keys, ts)):
            desc = f"{k} {t['what']} skew={t['skew']}"
            exp = E.NOT_IMPLEMENTED if t["skew"] else codes[t["verdict"]]
            self._outcome(i, desc, ecs[i], exp)
            if exp != E.OK:
                assert not self.cl.client.object_exists(k), f"{self.where(i, desc)}: a refused put was stored"
                continue
            _, ds = placed(t["table"], t["page"], 0, t["rw"], t["rp"], t["n"])
            x = host[ds]
            self.objs[k] = dm.Obj(_pack_model(x, w), "BBH64", reps, None, x, w) if fp8 else dm.Obj(x, algo, reps, None)
            self.blocks[k] = (t["page"], t["rw"], len(t["outer"]), t["ids"].size)
            self.outcomes["blocks put rebased"] += any(len(shs) > 1 for shs in self.shards(k))

    def get_blocks(self, fp8=False):
        bb, rng, E = self.bb, self.rng, self.bb.ErrorCode
        codes = {0: E.OK, 1: E.VALUE_OUT_OF_RANGE, 2: E.INVALID_ARGUMENT}
        keys = [k for k in self.pick(fp8, int(rng.integers(1, 5)), gone=0.2) if k in self.blocks]
        if not keys:
            return
        gw = str(rng.choice(WIDES)) if fp8 else None
        gb = WB[gw] if fp8 else 1
        per = 16 // gb
        ar = Arena(rng)
        specs = []
        for k in keys:
            page, rw, n_outer, n_ids = self.blocks[k]
            o = self.objs.get(k)
            rp = rw + per * int(rng.choice([1, 2, int(rng.integers(1, 24))])) if rw else 0
            stride = -(-extent(page, rw, rp) // per) * per + per * int(rng.choice([0, 1, 3]))
            n_blocks = n_ids + int(rng.integers(0, 16))
            skew = rng.random() < 0.15
            # duplicates drawn twice as often: they are the refusals only gets have
            refuse = None if skew or rng.random() < 0.6 else str(rng.choice(REFUSALS_GET + ["dup", "dup-ends", "dup-sel"]))
            partial = rng.random() < 0.4 or refuse in ("sel-high", "dup-sel")
            m = int(rng.integers(1, n_ids + 1)) if partial else n_ids
            if refuse in ("dup", "dup-ends", "dup-sel") and n_ids > 1:
                m = max(m, 2)
            dt = np.int32 if rng.random() < 0.5 else np.int64
            ids = rng.permutation(n_blocks)[:m].astype(np.int64)
            sel = rng.permutation(n_ids)[:m].astype(np.int64) if partial else None
            if refuse in ("high", "dup+high"):
                ids[int(rng.integers(0, m))] = n_blocks
            elif refuse == "neg":
                ids[int(rng.integers(0, m))] = -1
            elif refuse == "huge":
                dt, ids[0] = np.int64, (1 << 32) + int(ids[0])
            elif refuse == "sel-high" and partial:
                sel[int(rng.integers(0, m))] = n_ids
            elif refuse in ("dup", "dup-ends") and m > 1:
                ids[-1] = ids[0]
            elif refuse == "dup-sel" and partial and m > 1:
                sel[-1] = sel[0]
            base = ar.take(n_outer * n_blocks * stride, mod=per)
            outer = [base + q * n_blocks * stride for q in range(n_outer)]
            verdict, table = resolve(outer, ids, n_blocks, stride, sel, n_ids if partial else 0, get=True)
            t = dict(outer=outer, ids=ids.astype(dt), sel=None if sel is None else sel.astype(dt), n_stored=n_ids if partial else 0,
                     n_blocks=n_blocks, stride=stride, page=page, rw=rw, rp=rp, off=0, n=n_outer * n_ids * page, table=table)
            specs.append((k, o, t, verdict, skew))
        out = torch.full((ar.total + 16,), WGUARD[gb] if fp8 else GUARD, dtype={1: torch.uint8, 2: torch.int16, 4: torch.int32}[gb], device="cuda")
        blocks = [device_blocks(bb, t, out.data_ptr() + (8 if skew else 0), scale=gb) for _, _, t, _, skew in specs]
        self.what = f"{'fp8 as ' + gw + ' ' if fp8 else ''}blocks get of {len(keys)}"
        write_ids([s[2] for s in specs])
        if fp8:
            ecs = self.cl.client.batch_get_device_fp8_blocks(keys, blocks, _stream(), wide=dm._mx(bb, gw))
        else:
            ecs, sizes = self.cl.client.batch_get_device_blocks(keys, blocks, _stream())
        torch.cuda.synchronize()
        got = out.cpu().numpy().view({1: np.uint8, 2: np.uint16, 4: np.uint32}[gb])
        want = np.full(got.size, WGUARD[gb] if fp8 else GUARD, dtype=got.dtype)
        items = []
        for i, (k, o, t, verdict, skew) in enumerate(specs):
            desc = (f"{k} page={t['page']} rows {t['rw']}/{t['rp']} slices={len(t['outer'])} ids={t['ids'].size}x{t['ids'].itemsize}B"
                    f"{'' if t['sel'] is None else f' sel of {t['n_stored']}'} verdict={verdict} skew={skew}")
            if o is None:
                exp = E.OBJECT_NOT_FOUND
            elif skew or (fp8 and not self._fp8_usable(k)) or (len(t["table"]) > 1 and (t["page"] * gb) % 16):
                exp = E.NOT_IMPLEMENTED  # no fused path: a page of another type may be no multiple of 16 bytes
            else:
                exp = codes[verdict]
                if exp == E.OK:
                    xs, ds = placed(t["table"], t["page"], 0, t["rw"], t["rp"], t["n"])
                    if fp8:
                        want[ds] = o.back(gw)[xs]
                        _same(got[ds], want[ds], gw, self.where(i, desc))
                        got[ds] = want[ds]
                        self.outcomes["cross-type read"] += gw != o.w
                    else:
                        want[ds] = o.data[xs]
                        assert sizes[i] == o.data.size, f"{self.where(i, desc)}: size {sizes[i]}"
                    self.outcomes["partial restore"] += t["sel"] is not None
            self._outcome(i, desc, ecs[i], exp)
            items.append(desc)
        self._check_cache(got, want, items)

    def put_fp8_blocks(self):
        self.put_blocks(fp8=True)

    def get_fp8_blocks(self):
        self.get_blocks(fp8=True)

    def remove(self):
        super().remove()
        for k in list(self.blocks):
            if k not in self.objs:
                del self.blocks[k]

    def run(self, steps):
        weights = np.array([3, 4, 3, 4, 2, 3, 2, 3, 1], dtype=float)
        first = ["put_rows", "put_blocks", "put_fp8_rows", "put_fp8_blocks"]
        for self.step in range(steps):
            op = first[self.step] if self.step < len(first) else OPS[int(self.rng.choice(len(OPS), p=weights / weights.sum()))]
            self.ops[op] += 1
            getattr(self, op)()
            self.check_all()


@pytest.mark.parametrize("seed", SEEDS)
def test_random_layout_client_sequences(bb, seed):
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id=f"t-layout-model-{seed}", dram_bytes=128 << 20, high_watermark=1.0, max_replicas=3)
    try:
        m = LayoutModel(bb, cl, seed)
        m.run(STEPS)
        print(f"\nseed {seed}: operations {dict(m.ops)}; outcomes {dict(m.outcomes)}")
        for o in ("OK", "NOT_IMPLEMENTED", "VALUE_OUT_OF_RANGE", "INVALID_ARGUMENT", "OBJECT_NOT_FOUND", "rows put staged",
                  "rows get staged", "blocks put rebased", "partial restore", "cross-type read"):
            assert m.outcomes[o] > 0, f"seed {seed}: no {o} outcome in {STEPS} steps: {dict(m.outcomes)}"
    finally:
        cl.stop()
