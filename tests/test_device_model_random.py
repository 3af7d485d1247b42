"""Seeded random operation sequences through the client's device API on a GpuRankCluster with three tiers, against a
host model of the store.

The cluster has an HBM slab, a pinned shared-memory DRAM pool (which the fused kernels reach over PCIe) and an NVMe pool
(which device gets reach only through the host-staged path); ttl 0 and watermark 1.0, so nothing moves on its own.  Each
step draws a byte put (plain, strided or paged source, 1-3 replicas, 1-2 workers per copy so that shard edges fall
mid-page, any algorithm), an fp8 put (plain, strided or paged source, of bf16, fp16 or fp32 drawn per call), a byte get
(whole, range, strided, into pages or into rows), an fp8 get (whole, range, strided, into pages or into rows, in a type
drawn per call, so that objects packed from one type are read as another), a tier move, a compaction of the HBM pool, a
corruption of one copy or of every copy of an object followed by gets of it through any of those calls, or a remove.
Batches mix keys of different steps, tiers and algorithms; caller pointers and pages are sometimes misaligned, some
strided gaps and pages are no multiple of 16 bytes, some page tables repeat a page, and some destinations are too small
or larger than the object.

The model predicts every item's error code from the documented rules of blackbird_client.h, written out here: byte gets
are staged, never refused, and a paged or scattered one is BUFFER_OVERFLOW when the object is larger than its pages or
rows (a shorter object fills them in order) and INVALID_ARGUMENT for page size 0; whether a byte item is fused or staged
follows SourcePages::coaligned / fused_get_aligned and SourceRows::fused_get_aligned on every shard of every copy, and
reachability; an fp8 get is NOT_IMPLEMENTED when its virtual base, row 0 or a page is misaligned, when a multi-row slice
or scatter has a gap that is no multiple of 16 bytes, or when the object is not one shard in HBM or DRAM, and
INVALID_ARGUMENT when the element count is not that of the rows or pages; CHECKSUM_MISMATCH only when every copy read is
corrupt; OBJECT_NOT_FOUND after a remove.  After every step it checks the result bytes and the guard bytes around and
between them, every copy's stored bytes and recorded digest (Store in test_device_path.py) and the client counters the
step moves (staged items, placement refreshes).

Models trusted: numpy slicing, with the SourcePages and SourceRows rules of test_xfer_random.py; bb.crc32c / bb.bbh64 /
bb.xxh3t64 (checked in test_common.py against golden values, _bbh64_numpy and python-xxhash); the exact MXFP8 models of
test_mxfp8_exhaustive.py (model_pack, model_unpack) and test_mxfp8_wide.py (model_pack_w, model_unpack_w), checked
there against torch."""
import collections
import math
import os

import numpy as np
import pytest
import torch

from test_device_path import Store, _counter, _ref
from test_mxfp8_exhaustive import model_pack, model_unpack, same_bits
from test_xfer_random import WB, WGUARD, WIDES, _pack_model, _same, _unpack_model, pages_at, rows_at

pytestmark = pytest.mark.gpu

MiB = 1 << 20
GUARD = 0xA5
GUARD16 = 0x5A5A
T = 16384
ALGOS = ["NONE", "CRC32C", "BBH64", "XXH3"]
SEEDS = [3, 17]
STEPS = 150 + int(os.environ.get("BB_RANDOM_ROUNDS", "0")) * 10
OPS = ["put", "put_fp8", "get", "get_fp8", "migrate", "compact", "corrupt", "remove", "put_paged", "get_paged", "get_scatter",
       "put_fp8_paged", "get_fp8_paged", "get_fp8_scatter"]


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need CUDA (marked gpu)")
    free, _ = torch.cuda.mem_get_info()
    if free < (2 << 30) + (512 << 20):
        pytest.skip(f"needs about 2 GiB of free device memory, {free >> 20} MiB free")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _cluster(cid, tmp_path):
    from blackbird_b200.parallel import GpuRankCluster

    return GpuRankCluster(slab_bytes=256 << 20, cluster_id=cid, dram_bytes=128 << 20, nvme_bytes=256 << 20,
                          nvme_path=str(tmp_path), high_watermark=1.0, max_replicas=3)


def _cfg(bb, algo, replicas, tier, workers=1):
    return bb.WorkerConfig(replication_factor=replicas, max_workers_per_copy=workers, ttl_ms=0,
                           checksum=getattr(bb.ChecksumAlgo, algo), preferred_classes=[getattr(bb.StorageClass, tier)])


def _bf16(rng, n):
    """bf16 patterns across many binades, block by block (no NaN or Inf)."""
    top = rng.integers(60, 200, n // 32)[:, None]
    e = np.clip(top - rng.integers(0, 10, (n // 32, 32)), 0, 254)
    return ((e << 7) | rng.integers(0, 128, (n // 32, 32)) | (rng.integers(0, 2, (n // 32, 32)) << 15)).reshape(-1).astype(np.uint16)


def _wide(rng, n, w):
    """n patterns of type w across many binades, block by block (no NaN or Inf); fp16 reaches its subnormals."""
    if w == "bf16":
        return _bf16(rng, n)
    field, lo, hi, mant = (10, 2, 31, 10) if w == "f16" else (23, 60, 200, 23)
    top = rng.integers(lo, hi, n // 32)[:, None]
    e = np.clip(top - rng.integers(0, 10, (n // 32, 32)), 0, hi - 1)
    bits = (e << field) | rng.integers(0, 1 << mant, (n // 32, 32)) | (rng.integers(0, 2, (n // 32, 32)) << (field + (5 if w == "f16" else 8)))
    return bits.reshape(-1).astype(np.uint16 if w == "f16" else np.uint32)


def _mx(bb, w):
    return {"bf16": bb.MxWide.BF16, "f16": bb.MxWide.F16, "f32": bb.MxWide.F32}[w]


def _starts(shs):
    return np.cumsum([0] + [sh.length for sh in shs])[:-1].tolist()


def pages_coaligned(addrs, page, off, length):
    """SourcePages{addrs, page}.rebase(off).coaligned(length), written out: every page that object bytes [off, off +
    length) touch has addr + (off % page) 16-byte aligned, and the page is a multiple of 16 when they touch several."""
    ph, k0 = off % page, off // page
    n = (length - 1 + ph) // page + 1 if length else 0
    if n > 1 and page % 16:
        return False
    return all((addrs[k0 + j] + ph) % 16 == 0 for j in range(n))


def pages_fused(addrs, page, off, length):
    """SourcePages::fused_get_aligned: as pages_coaligned, and no table of several pages with page % 16 != 0."""
    return not (len(addrs) > 1 and page % 16) and pages_coaligned(addrs, page, off, length)


def rows_fused(dst, width, pitch, rows, off):
    """SourceRows::fused_get_aligned for the rows of a scattered get, from object byte off: a gap that is a multiple of 16
    and the rows co-aligned from where the shard starts."""
    if rows > 1 and width < pitch:
        return (pitch - width) % 16 == 0 and (dst + off // width * pitch + off % width) % 16 == 0
    return (dst + off) % 16 == 0


class Obj:
    """The model of one object: its bytes (a packed object's packed bytes), algorithm, copies and tier; a packed object's
    source patterns x and their type w."""

    def __init__(self, data, algo, copies, tier, x=None, w="bf16"):
        self.data, self.algo, self.copies, self.tier, self.x, self.w = data, algo, copies, tier, x, w
        self.flips = set()  # (copy, shard) corrupt right now
        self._back = {}

    def back(self, w):
        """What an fp8 get of type w returns: the unpack of the packed bytes in that type."""
        if w not in self._back:
            self._back[w] = _unpack_model(self.data, self.x.size, w)
        return self._back[w]

    @property
    def fp8(self):
        return self.x is not None


class Model:
    def __init__(self, bb, cl, seed):
        self.bb, self.cl, self.seed = bb, cl, seed
        self.rng = np.random.default_rng(seed)
        self.store = Store(bb, cl)
        self.objs, self.gone, self.next = {}, set(), 0
        self.ops, self.outcomes = collections.Counter(), collections.Counter()
        self.step, self.what = 0, ""

    def where(self, i=None, desc=""):
        return f"seed {self.seed} step {self.step} ({self.what})" + ("" if i is None else f" item {i} [{desc}]")

    def counter(self, name):
        return _counter(self.cl.client, name)

    # ------------------------------------------------------------------------------------------------ checks

    def shards(self, key):
        return [list(cp.shards) for cp in self.cl.client.get_workers(key)]

    def fabric(self, sh):
        """Whether the fused kernels reach a shard: HBM, or the mapped DRAM pool over PCIe; NVMe only through the host."""
        return sh.storage_class in (self.bb.StorageClass.RAM_GPU, self.bb.StorageClass.RAM_CPU)

    def check_copies(self, key):
        """Every copy of a live object holds the model's bytes (read back from HBM or DRAM) and carries the model's digest
        of them; after a move every shard is on the target tier.  Where a put places copies and stripes is the Keystone's
        choice: with three pools on one worker, replicas and stripes spread over the tiers."""
        o = self.objs[key]
        algo = "BBH64" if o.fp8 else o.algo
        placed = self.shards(key)
        assert len(placed) == o.copies, f"{self.where()}: {key} has {len(placed)} copies, want {o.copies}"
        ref = _ref(self.bb, algo)
        for c, shs in enumerate(placed):
            off = 0
            for s, sh in enumerate(shs):
                if o.tier is not None:
                    assert sh.storage_class == getattr(self.bb.StorageClass, o.tier), f"{self.where()}: {key} copy {c} on {sh.storage_class}, want {o.tier}"
                blob = o.data[off:off + sh.length]
                assert sh.checksum == ref(blob), f"{self.where()}: {key} copy {c} shard {s}: recorded digest"
                if self.fabric(sh):
                    assert self.store.stored(sh) == blob.tobytes(), f"{self.where()}: {key} copy {c} shard {s}: stored bytes"
                off += sh.length
            assert off == o.data.size, f"{self.where()}: {key} copy {c} holds {off} bytes"

    def check_all(self):
        for k in self.objs:
            self.check_copies(k)

    # ------------------------------------------------------------------------------------------------ operations

    def new_key(self):
        self.next += 1
        return f"s{self.seed}/k{self.next}"

    def pick(self, fp8, count, gone=0.0):
        keys = [k for k, o in self.objs.items() if o.fp8 == fp8]
        out = [str(self.rng.choice(keys)) for _ in range(count)] if keys else []
        if self.gone and self.rng.random() < gone:
            out.append(str(self.rng.choice(sorted(self.gone))))
        return out

    def put(self):
        bb, rng = self.bb, self.rng
        count = int(rng.integers(1, 6))
        algo, reps, workers = ALGOS[int(rng.integers(0, 4))], int(rng.integers(1, 4)), int(rng.integers(1, 3))
        tier = str(rng.choice(["RAM_GPU", "RAM_CPU"]))
        strided = rng.random() < 0.5
        self.what = f"put{' strided' if strided else ''} of {count}, {algo}, {reps} replicas, {workers} workers per copy, {tier}"
        keys = [self.new_key() for _ in range(count)]
        shapes = []  # (width, pitch, rows) of the source
        for _ in keys:
            n = int(rng.choice([int(rng.integers(1, 4097)), int(rng.integers(4097, 3 * T)), int(rng.integers(3 * T, 300000))]))
            if strided:
                width = int(rng.integers(1, min(n, 4000) + 1))
                pitch = width + int(rng.choice([0, 16 * int(rng.integers(1, 50)), int(rng.integers(1, 300))]))
                shapes.append((width, pitch, max(1, n // width)))
            else:
                shapes.append((n, n, 1))
        extents = [(r - 1) * p + w for w, p, r in shapes]
        offs, o = [], 0
        for e in extents:
            o = (o + 15) // 16 * 16 + (8 if rng.random() < 0.2 else 0)  # some sources misaligned: staged
            offs.append(o)
            o += e + 64
        src = torch.empty(o + 64, dtype=torch.uint8, device="cuda")
        bb.random_fill(src.data_ptr(), src.numel(), int(rng.integers(1, 1 << 40)), _stream())
        host = src.cpu().numpy()
        cfg = _cfg(bb, algo, reps, tier, workers)
        if strided:
            ecs = self.cl.client.batch_put_device_strided(keys, [src.data_ptr() + x for x in offs], [s[0] for s in shapes],
                                                          [s[1] for s in shapes], [s[2] for s in shapes], cfg, _stream())
        else:
            ecs = self.cl.client.batch_put_device(keys, [src.data_ptr() + x for x in offs], [s[0] for s in shapes], cfg, _stream())
        assert ecs == [bb.ErrorCode.OK] * count, f"{self.where()}: {ecs}"
        for k, x, (w, p, r) in zip(keys, offs, shapes):
            data = np.concatenate([host[x + i * p:x + i * p + w] for i in range(r)])
            self.objs[k] = Obj(data, algo, reps, None)

    def put_fp8(self):
        bb, rng = self.bb, self.rng
        count = int(rng.integers(1, 5))
        # one copy, on the tier asked for: further replicas may be placed on NVMe, which an fp8 put cannot write
        reps, tier, w = 1, str(rng.choice(["RAM_GPU", "RAM_CPU"])), str(rng.choice(WIDES))
        strided = rng.random() < 0.5
        self.what = f"fp8 put{' strided' if strided else ''} of {count}, {w}, {tier}"
        keys = [self.new_key() for _ in range(count)]
        shapes, xs, srcs = [], [], []
        for _ in keys:
            n = 32 * int(rng.choice([int(rng.integers(1, 200)), int(rng.integers(T // 32 - 1, T // 32 + 2)), int(rng.integers(T // 32, 4 * T // 32))]))
            if strided:
                width = 32 * int(rng.integers(1, 9))
                pitch = width + 8 * int(rng.integers(0, 20))
                rows = max(1, n // width)
            else:
                width, pitch, rows = n, n, 1
            x = _wide(rng, width * rows, w)
            buf = np.full((rows - 1) * pitch + width + 8, {"bf16": 0x7FC0, "f16": 0x7E00, "f32": 0x7FC00000}[w], dtype=x.dtype)  # NaN in the gaps
            for i in range(rows):
                buf[i * pitch:i * pitch + width] = x[i * width:(i + 1) * width]
            srcs.append(torch.from_numpy(buf.view(np.uint8)).cuda())
            shapes.append((width, pitch, rows))
            xs.append(x)
        cfg = _cfg(bb, "BBH64", reps, tier)
        ptrs = [s.data_ptr() for s in srcs]
        if strided:
            ecs = self.cl.client.batch_put_device_fp8_strided(keys, ptrs, [s[0] for s in shapes], [s[1] for s in shapes],
                                                              [s[2] for s in shapes], cfg, _stream(), wide=_mx(bb, w))
        else:
            ecs = self.cl.client.batch_put_device_fp8(keys, ptrs, [x.size for x in xs], cfg, _stream(), wide=_mx(bb, w))
        assert ecs == [bb.ErrorCode.OK] * count, f"{self.where()}: {ecs}"
        torch.cuda.synchronize()
        for k, x in zip(keys, xs):
            self.objs[k] = Obj(_pack_model(x, w), "BBH64", reps, tier, x, w)

    def _byte_shape(self, o):
        """(kind, offset, width, pitch, rows) of a byte get of object o: whole, range or strided."""
        rng, n = self.rng, o.data.size
        kind = str(rng.choice(["whole", "range", "strided"]))
        if kind == "whole":
            return kind, 0, n, n, 1
        off = int(rng.integers(0, n))
        if kind == "range":
            return kind, off, int(rng.integers(1, n - off + 1)), 0, 1
        width = int(rng.integers(1, min(n - off, 3000) + 1))
        pitch = width + int(rng.choice([0, 8, 16, 16 * int(rng.integers(1, 40)), int(rng.integers(1, 200))]))
        rows = 1 + (n - off - width) // pitch if pitch else 1
        return kind, off, width, pitch, int(rng.integers(1, rows + 1))

    def reads(self, key, off, width, pitch, rows):
        """Per copy, the (index, start, shard) of every shard a byte get of these rows reads: a whole or range get every
        shard its bytes overlap, a strided get every shard that holds a byte of a row."""
        out = []
        for shs in self.shards(key):
            start, got = 0, []
            for s, sh in enumerate(shs):
                if any(off + r * pitch < start + sh.length and off + r * pitch + width > start for r in range(rows)):
                    got.append((s, start, sh))
                start += sh.length
            out.append(got)
        return out

    def staged(self, key, ptr, off, width, pitch, rows):
        """The client's documented rule: a byte get takes the fused kernel only if its virtual base ptr - off is 16-byte
        aligned at the start of every shard of every copy (for a strided get, of the shards it reads, and its gap is a
        multiple of 16 when it has several rows) and some copy has every shard the get reads in HBM or DRAM."""
        strided = rows > 1 and width < pitch
        if strided and (pitch - width) % 16:
            return True
        if strided:
            per_copy = [[start for _, start, _ in c] for c in self.reads(key, off, width, pitch, rows)]
        else:
            per_copy = [list(np.cumsum([0] + [sh.length for sh in shs])[:-1]) for shs in self.shards(key)]
        if any((ptr - off + int(start)) % 16 for c in per_copy for start in c):
            return True
        return not any(all(self.fabric(sh) for _, _, sh in c) for c in self.reads(key, off, width, pitch, rows))

    def mismatch(self, key, o, off, width, pitch, rows):
        """CHECKSUM_MISMATCH: every copy has a corrupt shard among those the get reads (an unchecked algorithm reads no
        corruption)."""
        if not o.flips or o.algo == "NONE":
            return False
        return all(any((c, s) in o.flips for s, _, _ in got) for c, got in enumerate(self.reads(key, off, width, pitch, rows)))

    def get(self, keys=None):
        bb, rng = self.bb, self.rng
        keys = keys or self.pick(False, int(rng.integers(1, 8)), gone=0.3)
        if not keys:
            return
        kinds = collections.Counter()
        items, o_ = [], 64
        for k in keys:
            o = self.objs.get(k)
            shape = ("range", 0, 100, 0, 1) if o is None else self._byte_shape(o)
            kinds[shape[0]] += 1
            size = shape[2] * shape[4]
            skew = 8 if rng.random() < 0.2 else int(rng.choice([0, 1, 3])) if rng.random() < 0.1 else 0
            region = (o_ + 15) // 16 * 16 + (shape[1] + skew) % 16  # virtual base aligned unless skewed
            items.append((k, o, shape, region))
            o_ = region + size + 48
        out = torch.full((o_ + 64,), GUARD, dtype=torch.uint8, device="cuda")
        p = out.data_ptr()
        self.what = f"byte get of {len(keys)}: {dict(kinds)}"
        # one call per shape: whole gets, range gets, strided gets
        ecs = {}
        st0, ref0, fo0 = self.counter("device_get_host_staged_total"), self.counter("get_placement_refresh_total"), self.counter("replica_failover_total")
        staged = 0
        for kind in ("whole", "range", "strided"):
            idx = [i for i, it in enumerate(items) if it[2][0] == kind]
            if not idx:
                continue
            ks = [items[i][0] for i in idx]
            ptrs = [p + items[i][3] for i in idx]
            if kind == "whole":
                got, sizes = self.cl.client.batch_get_device(ks, ptrs, [items[i][2][2] + 16 for i in idx], _stream())
            elif kind == "range":
                got = self.cl.client.batch_get_device_range(ks, ptrs, [items[i][2][1] for i in idx], [items[i][2][2] for i in idx], _stream())
            else:
                got = self.cl.client.batch_get_device_strided(ks, ptrs, [items[i][2][1] for i in idx], [items[i][2][2] for i in idx],
                                                              [items[i][2][3] for i in idx], [items[i][2][4] for i in idx], _stream())
            for i, ec in zip(idx, got):
                ecs[i] = ec
        torch.cuda.synchronize()
        want = np.full(out.numel(), GUARD, dtype=np.uint8)
        mismatches = 0
        for i, (k, o, (kind, off, w, pitch, rows), region) in enumerate(items):
            desc = f"{k} {kind} off={off} width={w} pitch={pitch} rows={rows} region%16={region % 16}"
            if o is None:
                exp = bb.ErrorCode.OBJECT_NOT_FOUND
            else:
                desc += f" n={o.data.size} {o.algo} tier={o.tier} x{o.copies}"
                bad_ = self.mismatch(k, o, off, w, pitch, rows)
                exp = bb.ErrorCode.CHECKSUM_MISMATCH if bad_ else bb.ErrorCode.OK
                # a get that fails on every copy is issued once more by the placement refresh
                staged += self.staged(k, p + region, off, w, pitch, rows) * (1 + bad_)
            assert ecs[i] == exp, f"{self.where(i, desc)}: {ecs[i]}, want {exp}"
            mismatches += exp == bb.ErrorCode.CHECKSUM_MISMATCH
            if exp == bb.ErrorCode.OK:
                rows_ = [o.data[off + r * pitch:off + r * pitch + w] for r in range(rows)]
                want[region:region + w * rows] = np.concatenate(rows_)
            self.outcomes[str(exp).split(".")[-1]] += 1
        got = out.cpu().numpy()
        for i, (k, o, (kind, off, w, pitch, rows), region) in enumerate(items):
            if ecs[i] == bb.ErrorCode.CHECKSUM_MISMATCH:  # the result of a failed get is unspecified, nothing around it
                want[region:region + w * rows] = got[region:region + w * rows]
        bad = np.nonzero(got != want)[0]
        if bad.size:
            first = int(bad[0])
            near = [(i, it[0], it[2]) for i, it in enumerate(items) if it[3] - 48 <= first < it[3] + it[2][2] * it[2][4] + 48]
            pytest.fail(f"{self.where()}: {bad.size} wrong bytes, first at {first}, near items {near}")
        assert self.counter("device_get_host_staged_total") - st0 == staged, f"{self.where()}: staged items"
        assert self.counter("get_placement_refresh_total") - ref0 == mismatches, f"{self.where()}: placement refreshes"
        staged_ok = sum(self.staged(it[0], p + it[3], *it[2][1:]) for i, it in enumerate(items) if ecs[i] == bb.ErrorCode.OK)
        self.outcomes["staged"] += staged_ok
        self.outcomes["fused"] += sum(1 for v in ecs.values() if v == bb.ErrorCode.OK) - staged_ok
        self.outcomes["fail-over"] += self.counter("replica_failover_total") - fo0

    def _fp8_shape(self, o):
        rng, n = self.rng, o.x.size
        kind = str(rng.choice(["whole", "range", "strided"]))
        if kind == "whole":
            return kind, 0, n, n, 1
        off = int(rng.integers(0, n))
        if kind == "range":
            return kind, off, int(rng.integers(1, n - off + 1)), 0, 1
        width = int(rng.integers(1, min(n - off, 2000) + 1))
        pitch = width + int(rng.choice([0, 4, 8, 8 * int(rng.integers(1, 30)), int(rng.integers(1, 100))]))
        rows = 1 + (n - off - width) // pitch
        return kind, off, width, pitch, int(rng.integers(1, rows + 1))

    def get_fp8(self, keys=None):
        bb, rng = self.bb, self.rng
        keys = keys or self.pick(True, int(rng.integers(1, 7)), gone=0.3)
        if not keys:
            return
        gw = str(rng.choice(WIDES))  # the type of the call: objects packed from any type are read into it
        gb, per = WB[gw], 16 // WB[gw]
        items, o_ = [], 64
        for k in keys:
            o = self.objs.get(k)
            shape = ("range", 0, 64, 0, 1) if o is None else self._fp8_shape(o)
            # misaligned ranges and slices fail alone (NOT_IMPLEMENTED); a whole tensor's pointer is the engine's to check
            skew = int(rng.choice([1, per // 2])) if rng.random() < 0.2 and shape[0] != "whole" else 0
            region = (o_ + per - 1) // per * per + (shape[1] + skew) % per  # element offset: virtual base aligned unless skewed
            items.append((k, o, shape, region, skew))
            o_ = region + shape[2] * shape[4] + 32
        out = torch.full((o_ + 64,), WGUARD[gb], dtype=torch.int16 if gb == 2 else torch.int32, device="cuda")
        p = out.data_ptr()
        self.what = f"fp8 get of {len(keys)} as {gw}"
        ecs = {}
        ref0, fo0 = self.counter("get_placement_refresh_total"), self.counter("replica_failover_total")
        for kind in ("whole", "range", "strided"):
            idx = [i for i, it in enumerate(items) if it[2][0] == kind]
            if not idx:
                continue
            ks = [items[i][0] for i in idx]
            ptrs = [p + gb * items[i][3] for i in idx]
            ns = [items[i][1].x.size if items[i][1] is not None else 64 for i in idx]
            if kind == "whole":
                got = self.cl.client.batch_get_device_fp8(ks, ptrs, ns, _stream(), wide=_mx(bb, gw))
            elif kind == "range":
                got = self.cl.client.batch_get_device_fp8_range(ks, ptrs, ns, [items[i][2][1] for i in idx], [items[i][2][2] for i in idx], _stream(),
                                                               wide=_mx(bb, gw))
            else:
                got = self.cl.client.batch_get_device_fp8_strided(ks, ptrs, ns, [items[i][2][1] for i in idx], [items[i][2][2] for i in idx],
                                                                  [items[i][2][3] for i in idx], [items[i][2][4] for i in idx], _stream(),
                                                                  wide=_mx(bb, gw))
            for i, ec in zip(idx, got):
                ecs[i] = ec
        torch.cuda.synchronize()
        written = np.zeros(out.numel(), dtype=bool)
        E = bb.ErrorCode
        mismatches = 0
        for i, (k, o, (kind, off, w, pitch, rows), region, skew) in enumerate(items):
            desc = f"{k} {kind} off={off} width={w} pitch={pitch} rows={rows} skew={skew}"
            if o is None:
                exp = E.OBJECT_NOT_FOUND
            else:
                desc += f" n={o.x.size} packed as {o.w} {o.tier} x{o.copies}"
                gap_bad = rows > 1 and w < pitch and (pitch - w) % per != 0
                usable = any(len(shs) == 1 and self.fabric(shs[0]) for shs in self.shards(k))
                # the whole-object call leaves alignment to the engine: its buffers here are always aligned
                if not usable or (kind != "whole" and (skew or gap_bad)):
                    exp = E.NOT_IMPLEMENTED
                elif self.mismatch(k, o, 0, o.data.size, o.data.size, 1):
                    exp = E.CHECKSUM_MISMATCH
                else:
                    exp = E.OK
            assert ecs[i] == exp, f"{self.where(i, desc)}: {ecs[i]}, want {exp}"
            mismatches += exp == E.CHECKSUM_MISMATCH
            if exp == E.CHECKSUM_MISMATCH:  # the result of a failed get is unspecified, nothing around it
                written[region:region + w * rows] = True
            if exp == E.OK:
                el = np.concatenate([np.arange(off + r * pitch, off + r * pitch + w) for r in range(rows)])
                written[region:region + el.size] = True
                _same(out[region:region + el.size].cpu().numpy(), o.back(gw)[el], gw, self.where(i, desc))
                self.outcomes["cross-type read"] += gw != o.w
            self.outcomes[str(exp).split(".")[-1]] += 1
            self.outcomes["fused"] += exp == E.OK
        got = out.cpu().numpy().view(np.uint16 if gb == 2 else np.uint32)
        bad = np.nonzero(~written & (got != WGUARD[gb]))[0]
        assert bad.size == 0, f"{self.where()}: {bad.size} elements written outside the results, first at {bad[:4].tolist()}"
        assert self.counter("get_placement_refresh_total") - ref0 == mismatches, f"{self.where()}: placement refreshes"
        self.outcomes["fail-over"] += self.counter("replica_failover_total") - fo0

    # ------------------------------------------------------------------------------------------------ pages and rows

    def put_staged(self, key, addrs, page):
        """The client's documented rule for a paged put: fused only if every shard of every copy is co-aligned with the
        pages (SourcePages::coaligned from the shard's start) and every shard is reachable by the fabric."""
        placed = self.shards(key)
        ok = all(pages_coaligned(addrs, page, off, sh.length) for shs in placed for off, sh in zip(_starts(shs), shs))
        return not ok or not all(self.fabric(sh) for shs in placed for sh in shs)

    def get_staged(self, key, aligned):
        """The rule of a whole-object get into pages or rows: fused only if aligned(off, length) holds for every shard of
        every copy and some copy has every shard in HBM or DRAM."""
        placed = self.shards(key)
        if not all(aligned(off, sh.length) for shs in placed for off, sh in zip(_starts(shs), shs)):
            return True
        return not any(all(self.fabric(sh) for sh in shs) for shs in placed)

    def put_paged(self):
        bb, rng = self.bb, self.rng
        count = int(rng.integers(1, 5))
        algo, reps, workers = ALGOS[int(rng.integers(0, 4))], int(rng.integers(1, 4)), int(rng.integers(1, 3))
        tier = str(rng.choice(["RAM_GPU", "RAM_CPU"]))
        self.what = f"paged put of {count}, {algo}, {reps} replicas, {workers} workers per copy, {tier}"
        keys = [self.new_key() for _ in range(count)]
        specs = []  # (page, pages, skew, repeats)
        for _ in keys:
            page = int(rng.choice([16, 48, 4096, T + 16, 32768 + 48, 16 * int(rng.integers(1, 300)), int(rng.integers(1, 5000)) | 1]))
            npg = 1 if page % 16 else int(rng.integers(1, max(2, min(200, 300000 // page)) + 1))
            specs.append((0 if rng.random() < 0.05 else page, npg, 8 if rng.random() < 0.15 else 0, npg > 1 and rng.random() < 0.2))
        slot = (max(max(s[0], 16) for s in specs) + 15) // 16 * 16 + 64
        src = torch.empty(sum(s[1] for s in specs) * slot + 64, dtype=torch.uint8, device="cuda")
        bb.random_fill(src.data_ptr(), src.numel(), int(rng.integers(1, 1 << 40)), _stream())
        host = src.cpu().numpy()
        free = list(rng.permutation(sum(s[1] for s in specs)))
        lists, datas = [], []
        for page, npg, skew, rep in specs:
            offs = [int(free.pop()) * slot + skew for _ in range(npg)]
            if rep:  # a page may repeat
                for j in rng.integers(0, npg, max(1, npg // 4)):
                    offs[int(j)] = offs[int(rng.integers(0, npg))]
            lists.append([src.data_ptr() + o for o in offs])
            datas.append(np.concatenate([host[o:o + page] for o in offs]) if page else None)
        st0 = self.counter("device_put_host_staged_total")
        ecs = self.cl.client.batch_put_device_paged(keys, lists, [s[0] for s in specs], _cfg(bb, algo, reps, tier, workers), _stream())
        staged = 0
        for i, (k, (page, npg, skew, rep), addrs, data) in enumerate(zip(keys, specs, lists, datas)):
            desc = f"{k} page={page} pages={npg} skew={skew} repeats={rep}"
            exp = bb.ErrorCode.INVALID_ARGUMENT if page == 0 else bb.ErrorCode.OK
            assert ecs[i] == exp, f"{self.where(i, desc)}: {ecs[i]}, want {exp}"
            self.outcomes[str(exp).split(".")[-1]] += 1
            if page:
                self.objs[k] = Obj(data, algo, reps, None)
                staged += self.put_staged(k, addrs, page)
        assert self.counter("device_put_host_staged_total") - st0 == staged, f"{self.where()}: staged items"
        self.outcomes["put staged"] += staged

    def _results(self, out, want, items):
        """Every result byte and every guard byte: `items` = (description, result offsets) per item."""
        got = out.cpu().numpy().view(want.dtype)
        bad = np.nonzero(got != want)[0]
        if bad.size:
            first = int(bad[0])
            near = [(i, d) for i, (d, ds) in enumerate(items) if ds.size and ds.min() - 64 <= first <= ds.max() + 64]
            pytest.fail(f"{self.where()}: {bad.size} wrong result or guard units, first at {first} (got {got[first]:#x}, "
                        f"want {want[first]:#x}), near items {near}")

    def get_paged(self, keys=None):
        bb, rng = self.bb, self.rng
        E = bb.ErrorCode
        keys = keys or self.pick(False, int(rng.integers(1, 6)), gone=0.3)
        if not keys:
            return
        specs, cur = [], 64
        for k in keys:
            o = self.objs.get(k)
            n = o.data.size if o else 100
            page = int(rng.choice([16, 48, 4096, T + 16, 32768 + 48, 16 * int(rng.integers(1, 100)) + 8]))
            npg = -(-n // page)
            r = rng.random()
            npg = npg - 1 if r < 0.1 else npg + int(rng.integers(1, 3)) if r < 0.3 else npg  # too few pages, or more than needed
            skew = 8 if rng.random() < 0.15 else 0
            stride = (page + 15) // 16 * 16 + 48
            offs = [cur + int(j) * stride + skew for j in rng.permutation(npg)]
            cur += npg * stride + 64
            specs.append((k, o, 0 if o is not None and offs and rng.random() < 0.05 else page, offs))  # page 0 with pages
        out = torch.full((cur + 64,), GUARD, dtype=torch.uint8, device="cuda")
        p = out.data_ptr()
        self.what = f"paged get of {len(keys)}"
        st0, ref0, fo0 = self.counter("device_get_host_staged_total"), self.counter("get_placement_refresh_total"), self.counter("replica_failover_total")
        ecs, sizes = self.cl.client.batch_get_device_paged(keys, [[p + a for a in s[3]] for s in specs], [s[2] for s in specs], _stream())
        torch.cuda.synchronize()
        want = np.full(out.numel(), GUARD, dtype=np.uint8)
        staged = mismatches = 0
        items = []
        for i, (k, o, page, offs) in enumerate(specs):
            desc = f"{k} page={page} pages={len(offs)} skew={offs[0] % 16 if offs else 0}"
            ds = np.zeros(0, dtype=np.int64)
            if o is None:
                exp = E.OBJECT_NOT_FOUND
            elif page == 0:
                exp = E.INVALID_ARGUMENT
            elif o.data.size > page * len(offs):
                exp = E.BUFFER_OVERFLOW
            else:
                desc += f" n={o.data.size} {o.algo} tier={o.tier} x{o.copies}"
                bad_ = self.mismatch(k, o, 0, o.data.size, o.data.size, 1)
                exp = E.CHECKSUM_MISMATCH if bad_ else E.OK
                addrs = [p + a for a in offs]
                staged += self.get_staged(k, lambda off, ln: pages_fused(addrs, page, off, ln)) * (1 + bad_)
                ds = pages_at(o.data.size, offs, page, 0)
                if exp == E.OK:
                    want[ds] = o.data
                    assert sizes[i] == o.data.size, f"{self.where(i, desc)}: size {sizes[i]}"
                    self.outcomes["paged fused"] += not self.get_staged(k, lambda off, ln: pages_fused(addrs, page, off, ln))
                else:
                    want[ds] = out[torch.from_numpy(ds).cuda()].cpu().numpy()  # unspecified, nothing around them
            assert ecs[i] == exp, f"{self.where(i, desc)}: {ecs[i]}, want {exp}"
            mismatches += exp == E.CHECKSUM_MISMATCH
            self.outcomes[str(exp).split(".")[-1]] += 1
            items.append((desc, ds))
        self._results(out, want, items)
        assert self.counter("device_get_host_staged_total") - st0 == staged, f"{self.where()}: staged items"
        assert self.counter("get_placement_refresh_total") - ref0 == mismatches, f"{self.where()}: placement refreshes"
        self.outcomes["fail-over"] += self.counter("replica_failover_total") - fo0

    def get_scatter(self, keys=None):
        bb, rng = self.bb, self.rng
        E = bb.ErrorCode
        keys = keys or self.pick(False, int(rng.integers(1, 6)), gone=0.3)
        if not keys:
            return
        specs, cur = [], 64
        for k in keys:
            o = self.objs.get(k)
            n = o.data.size if o else 100
            width = int(rng.integers(1, min(n, 4000) + 1))
            pitch = width + int(rng.choice([0, 16, 16 * int(rng.integers(1, 40)), int(rng.integers(1, 200))]))
            rows = -(-n // width)
            r = rng.random()
            rows = rows - 1 if r < 0.1 else rows + int(rng.integers(1, 3)) if r < 0.25 else rows
            skew = 8 if rng.random() < 0.15 else int(rng.choice([0, 1, 3])) if rng.random() < 0.1 else 0
            at = (cur + 15) // 16 * 16 + skew
            cur = at + max(rows - 1, 0) * pitch + width + 64
            specs.append((k, o, width, pitch, rows, at))
        out = torch.full((cur + 64,), GUARD, dtype=torch.uint8, device="cuda")
        p = out.data_ptr()
        self.what = f"scattered get of {len(keys)}"
        st0, ref0, fo0 = self.counter("device_get_host_staged_total"), self.counter("get_placement_refresh_total"), self.counter("replica_failover_total")
        ecs, sizes = self.cl.client.batch_get_device_scatter(keys, [p + s[5] for s in specs], [s[2] for s in specs], [s[3] for s in specs],
                                                             [s[4] for s in specs], _stream())
        torch.cuda.synchronize()
        want = np.full(out.numel(), GUARD, dtype=np.uint8)
        staged = mismatches = 0
        items = []
        for i, (k, o, width, pitch, rows, at) in enumerate(specs):
            desc = f"{k} width={width} pitch={pitch} rows={rows} at%16={at % 16}"
            ds = np.zeros(0, dtype=np.int64)
            if o is None:
                exp = E.OBJECT_NOT_FOUND
            elif o.data.size > rows * width:
                exp = E.BUFFER_OVERFLOW
            else:
                desc += f" n={o.data.size} {o.algo} tier={o.tier} x{o.copies}"
                bad_ = self.mismatch(k, o, 0, o.data.size, o.data.size, 1)
                exp = E.CHECKSUM_MISMATCH if bad_ else E.OK
                staged += self.get_staged(k, lambda off, ln: rows_fused(p + at, width, pitch, rows, off)) * (1 + bad_)
                ds = at + rows_at(o.data.size, pitch if rows > 1 else width, width, 0)
                if exp == E.OK:
                    want[ds] = o.data
                    assert sizes[i] == o.data.size, f"{self.where(i, desc)}: size {sizes[i]}"
                else:
                    want[ds] = out[torch.from_numpy(ds).cuda()].cpu().numpy()  # unspecified, nothing around them
            assert ecs[i] == exp, f"{self.where(i, desc)}: {ecs[i]}, want {exp}"
            mismatches += exp == E.CHECKSUM_MISMATCH
            self.outcomes[str(exp).split(".")[-1]] += 1
            items.append((desc, ds))
        self._results(out, want, items)
        assert self.counter("device_get_host_staged_total") - st0 == staged, f"{self.where()}: staged items"
        assert self.counter("get_placement_refresh_total") - ref0 == mismatches, f"{self.where()}: placement refreshes"
        self.outcomes["fail-over"] += self.counter("replica_failover_total") - fo0

    def put_fp8_paged(self):
        bb, rng = self.bb, self.rng
        E = bb.ErrorCode
        count = int(rng.integers(1, 4))
        tier, w = str(rng.choice(["RAM_GPU", "RAM_CPU"])), str(rng.choice(WIDES))
        b, per = WB[w], 16 // WB[w]
        self.what = f"fp8 paged put of {count}, {w}, {tier}"
        keys = [self.new_key() for _ in range(count)]
        specs, cur = [], 16
        for _ in keys:
            page = int(rng.choice([per, 3 * per, 32, 5 * per, 8 * per * int(rng.integers(1, 40)), per * int(rng.integers(1, 50)) + per // 2]))
            npg = 32 // math.gcd(page, 32) * int(rng.integers(1, max(2, 6000 // page)))  # a whole number of MX blocks
            if rng.random() < 0.08:
                npg += 1  # unless that makes a partial block
            skew = b if rng.random() < 0.12 else 0  # one page off 16-byte alignment
            stride = (page * b + 15) // 16 * 16 + 32
            offs = [cur + int(j) * stride for j in rng.permutation(npg)]
            if skew:
                offs[int(rng.integers(0, npg))] += skew
            cur += npg * stride + 32
            specs.append((page, offs))
        buf = np.full(cur + 64, GUARD, dtype=np.uint8)
        xs = []
        for page, offs in specs:
            x = _wide(rng, page * len(offs) // 32 * 32 + 32, w)[:page * len(offs)]
            buf[pages_at(x.size * b, offs, page * b, 0)] = x.view(np.uint8)
            xs.append(x)
        src = torch.from_numpy(buf).cuda()
        lists = [[src.data_ptr() + o for o in offs] for _, offs in specs]
        ecs = self.cl.client.batch_put_device_fp8_paged(keys, lists, [s[0] for s in specs], _cfg(bb, "BBH64", 1, tier), _stream(),
                                                        wide=_mx(bb, w))
        torch.cuda.synchronize()
        for i, (k, (page, offs), x) in enumerate(zip(keys, specs, xs)):
            desc = f"{k} page={page} pages={len(offs)} n={x.size}"
            if x.size % 32:
                exp = E.INVALID_ARGUMENT
            elif not pages_coaligned(lists[i], page * b, 0, x.size * b):
                exp = E.NOT_IMPLEMENTED
            else:
                exp = E.OK
                self.objs[k] = Obj(_pack_model(x, w), "BBH64", 1, tier, x, w)
            assert ecs[i] == exp, f"{self.where(i, desc)}: {ecs[i]}, want {exp}"
            self.outcomes[str(exp).split(".")[-1]] += 1

    def _fp8_usable(self, k):
        return any(len(shs) == 1 and self.fabric(shs[0]) for shs in self.shards(k))

    def get_fp8_paged(self, keys=None, scatter=False):
        """Gets of packed objects into pages (or, scatter=True, into rows), in a type drawn per call."""
        bb, rng = self.bb, self.rng
        E = bb.ErrorCode
        keys = keys or self.pick(True, int(rng.integers(1, 5)), gone=0.3)
        if not keys:
            return
        gw = str(rng.choice(WIDES))
        gb, per = WB[gw], 16 // WB[gw]
        specs, cur = [], 16  # in elements
        for k in keys:
            o = self.objs.get(k)
            n = o.x.size if o else 64
            skew = int(rng.choice([1, per // 2])) if rng.random() < 0.15 else 0
            if scatter:
                width = 32 * int(rng.choice([d for d in (1, 2, 3, 4, 8, 16) if (n // 32) % d == 0]))
                width = n if rng.random() < 0.1 else width
                pitch = width + int(rng.choice([0, per, per * int(rng.integers(1, 30)), int(rng.integers(1, 100))]))
                rows = n // width - (1 if o is not None and n > width and rng.random() < 0.05 else 0)
                at = (cur + per - 1) // per * per + skew
                cur = at + max(rows - 1, 0) * pitch + width + 32
                specs.append((k, o, (width, pitch, rows), at))
            else:
                page = int(rng.choice([d for d in (per, 3 * per, 32, 5 * per, 8 * per, 40 * per, n) if n % d == 0]))
                if o is not None and rng.random() < 0.08:
                    page += 1  # pages * page may no longer be the object's element count
                npg = -(-n // page)
                stride = (page + per - 1) // per * per + 2 * per
                offs = [cur + int(j) * stride for j in rng.permutation(npg)]
                if skew:
                    offs[int(rng.integers(0, npg))] += skew
                cur += npg * stride + 32
                specs.append((k, o, page, offs))
        out = torch.full((cur + 64,), WGUARD[gb], dtype=torch.int16 if gb == 2 else torch.int32, device="cuda")
        p = out.data_ptr()
        self.what = f"fp8 {'scattered' if scatter else 'paged'} get of {len(keys)} as {gw}"
        ref0, fo0 = self.counter("get_placement_refresh_total"), self.counter("replica_failover_total")
        ns = [s[1].x.size if s[1] is not None else 64 for s in specs]
        if scatter:
            ecs = self.cl.client.batch_get_device_fp8_scatter(keys, [p + gb * s[3] for s in specs], ns, [s[2][0] for s in specs],
                                                              [s[2][1] for s in specs], [s[2][2] for s in specs], _stream(), wide=_mx(bb, gw))
        else:
            ecs = self.cl.client.batch_get_device_fp8_paged(keys, [[p + gb * a for a in s[3]] for s in specs], [s[2] for s in specs], _stream(),
                                                            wide=_mx(bb, gw))
        torch.cuda.synchronize()
        got = out.cpu().numpy().view(np.uint16 if gb == 2 else np.uint32)
        written = np.zeros(got.size, dtype=bool)
        mismatches = 0
        for i, (k, o, shape, at) in enumerate(specs):
            desc = f"{k} {'rows (width, pitch, rows)' if scatter else 'page'}={shape} {'at' if scatter else 'pages'}={at if scatter else len(at)}"
            if o is None:
                exp = E.OBJECT_NOT_FOUND
            else:
                n = o.x.size
                desc += f" n={n} packed as {o.w} {o.tier}"
                if scatter:
                    width, pitch, rows = shape
                    ds = at + rows_at(n, pitch if rows > 1 else width, width, 0)
                    count_ok = rows * width == n
                    aligned = (p + gb * at) % 16 == 0 and not (rows > 1 and width < pitch and (pitch - width) % per)
                else:
                    ds = pages_at(n, at, shape, 0) if len(at) * shape >= n else np.zeros(0, dtype=np.int64)
                    count_ok = len(at) * shape == n
                    addrs = [p + gb * a for a in at]
                    aligned = not (len(at) > 1 and (shape * gb) % 16) and pages_coaligned(addrs, shape * gb, 0, n * gb)
                if not count_ok:
                    exp = E.INVALID_ARGUMENT
                elif not self._fp8_usable(k) or not aligned:
                    exp = E.NOT_IMPLEMENTED
                elif self.mismatch(k, o, 0, o.data.size, o.data.size, 1):
                    exp = E.CHECKSUM_MISMATCH
                    written[ds] = True  # unspecified, nothing around them
                else:
                    exp = E.OK
                    written[ds] = True
                    _same(got[ds], o.back(gw), gw, self.where(i, desc))
                    self.outcomes["cross-type read"] += gw != o.w
            assert ecs[i] == exp, f"{self.where(i, desc)}: {ecs[i]}, want {exp}"
            mismatches += exp == E.CHECKSUM_MISMATCH
            self.outcomes[str(exp).split(".")[-1]] += 1
            self.outcomes["fused"] += exp == E.OK
        bad = np.nonzero(~written & (got != WGUARD[gb]))[0]
        assert bad.size == 0, f"{self.where()}: {bad.size} elements written outside the results, first at {bad[:4].tolist()}"
        assert self.counter("get_placement_refresh_total") - ref0 == mismatches, f"{self.where()}: placement refreshes"
        self.outcomes["fail-over"] += self.counter("replica_failover_total") - fo0

    def get_fp8_scatter(self, keys=None):
        self.get_fp8_paged(keys, scatter=True)

    def migrate(self):
        keys = [k for k in self.objs]
        if not keys:
            return
        k = str(self.rng.choice(keys))
        tier = str(self.rng.choice(["RAM_GPU", "RAM_CPU", "NVME"]))
        self.what = f"migrate {k} from {self.objs[k].tier} to {tier}"
        assert self.cl.client.migrate(k, getattr(self.bb.StorageClass, tier)) == self.bb.ErrorCode.OK, self.where()
        self.objs[k].tier = tier

    def compact(self):
        self.what = "compact hbm0"
        self.cl.client.keystone().compact_pool("hbm0")

    def corrupt(self):
        """Flip a byte of one copy (or of every copy) of an object, get it through every shape that reads it, restore."""
        rng = self.rng
        keys = [k for k, o in self.objs.items() if o.algo != "NONE" and all(self.fabric(sh) for shs in self.shards(k) for sh in shs)]
        if not keys:
            return
        everyone = rng.random() < 0.5
        replicated = [k for k in keys if self.objs[k].copies > 1]
        if not everyone and replicated and rng.random() < 0.7:  # one corrupt copy of several: the gets fail over
            keys = replicated
        k = str(rng.choice(keys))
        o = self.objs[k]
        placed = self.shards(k)
        flips = []
        for c, shs in enumerate(placed):
            if c and not everyone:
                break
            s = int(rng.integers(0, len(shs)))
            if shs[s].length:
                flips.append((c, s, int(rng.integers(0, shs[s].length))))
        self.what = f"corrupt {'every copy' if everyone else 'one copy'} of {k} (x{o.copies})"
        for c, s, pos in flips:
            self.store.flip(placed[c][s], pos)
        o.flips = {(c, s) for c, s, _ in flips}
        others = self.pick(o.fp8, 2)
        try:
            # a get of a shape drawn anew each time, then a get into pages or into rows
            calls = [self.get_fp8, self.get_fp8_paged, self.get_fp8_scatter] if o.fp8 else [self.get, self.get_paged, self.get_scatter]
            calls[0]([k] + others)
            calls[int(rng.integers(1, 3))]([k] + others)
        finally:
            for c, s, pos in flips:
                self.store.flip(placed[c][s], pos)
            o.flips = set()

    def remove(self):
        keys = list(self.objs)
        if not keys:
            return
        ks = [str(k) for k in self.rng.choice(keys, min(len(keys), int(self.rng.integers(1, 3))), replace=False)]
        self.what = f"remove {ks}"
        assert self.cl.client.batch_remove(ks) == [self.bb.ErrorCode.OK] * len(ks), self.where()
        for k in ks:
            del self.objs[k]
            self.gone.add(k)

    def run(self, steps):
        weights = np.array([3, 2, 4, 4, 2, 1, 3, 1, 2, 3, 3, 2, 2, 2], dtype=float)
        for self.step in range(steps):
            op = OPS[int(self.rng.choice(len(OPS), p=weights / weights.sum()))] if self.step >= 4 else ["put", "put_fp8"][self.step % 2]
            self.ops[op] += 1
            getattr(self, op)()
            self.check_all()


@pytest.mark.parametrize("seed", SEEDS)
def test_random_operation_sequences(bb, tmp_path, seed):
    cl = _cluster(f"t-model-{seed}", tmp_path)
    try:
        m = Model(bb, cl, seed)
        m.run(STEPS)
        print(f"\nseed {seed}: operations {dict(m.ops)}; outcomes {dict(m.outcomes)}")
        for o in ("fused", "staged", "NOT_IMPLEMENTED", "CHECKSUM_MISMATCH", "fail-over", "OBJECT_NOT_FOUND", "BUFFER_OVERFLOW",
                  "INVALID_ARGUMENT", "cross-type read", "paged fused", "put staged"):
            assert m.outcomes[o] > 0, f"seed {seed}: no {o} outcome in {STEPS} steps: {dict(m.outcomes)}"
    finally:
        cl.stop()


def test_fp8_gets_refresh_placements_and_follow_moves(bb, tmp_path):
    """The placement refresh of the fused-MXFP8 gets on the GPU: the only copy of a packed object corrupt, each of the three
    fp8 gets reports CHECKSUM_MISMATCH after exactly one refresh; once restored, the object is read from every placement
    a move or a compaction gives it: HBM, DRAM over PCIe, NVMe (NOT_IMPLEMENTED: no fused path) and HBM again."""
    cl = _cluster("t-model-refresh", tmp_path)
    try:
        E = bb.ErrorCode
        rng = np.random.default_rng(1)
        n = 3 * T + 96
        x = _bf16(rng, n)
        back = model_unpack(model_pack(x), n)
        src = torch.from_numpy(x.view(np.int16).copy()).cuda()
        filler = torch.empty(4 * MiB, dtype=torch.uint8, device="cuda")
        cfg = _cfg(bb, "BBH64", 1, "RAM_GPU")
        # a filler below the object, removed later, so that compaction has to move it
        assert cl.client.batch_put_device(["filler"], [filler.data_ptr()], [filler.numel()], cfg, _stream()) == [E.OK]
        assert cl.client.batch_put_device_fp8(["t"], [src.data_ptr()], [n], cfg, _stream()) == [E.OK]
        store = Store(bb, cl)
        out = torch.full((n + 64,), GUARD16, dtype=torch.int16, device="cuda")
        p = out.data_ptr() + 64  # element 32: 16-byte aligned
        rows = (40, 200, 1000, 30)  # offset, width, pitch, rows (gap of 800 elements)
        rel = np.concatenate([np.arange(40 + r * 1000, 240 + r * 1000) for r in range(30)])
        gets = {"whole": (lambda: cl.client.batch_get_device_fp8(["t"], [p], [n], _stream()), np.arange(n)),
                "range": (lambda: cl.client.batch_get_device_fp8_range(["t"], [p], [n], [T - 8], [5000], _stream()), np.arange(T - 8, T + 4992)),
                "strided": (lambda: cl.client.batch_get_device_fp8_strided(["t"], [p], [n], [rows[0]], [rows[1]], [rows[2]], [rows[3]], _stream()), rel)}

        def read_all(expect, what):
            for name, (call, el) in gets.items():
                out.fill_(GUARD16)
                r0 = _counter(cl.client, "get_placement_refresh_total")
                assert call() == [expect], (what, name)
                assert _counter(cl.client, "get_placement_refresh_total") == r0 + (expect == E.CHECKSUM_MISMATCH), (what, name)
                torch.cuda.synchronize()
                got = out.cpu().numpy().view(np.uint16)
                if expect == E.OK:
                    same_bits(got[32:32 + el.size], back[el], "bf16", f"{what}: {name}")
                    assert bool((got[:32] == GUARD16).all()) and bool((got[32 + el.size:] == GUARD16).all()), (what, name)
                else:
                    assert expect == E.CHECKSUM_MISMATCH or bool((got == GUARD16).all()), (what, name)

        read_all(E.OK, "HBM")
        sh = cl.client.get_workers("t")[0].shards[0]
        store.flip(sh, n + 7)  # a scale byte
        read_all(E.CHECKSUM_MISMATCH, "the only copy corrupt")
        store.flip(sh, n + 7)
        before = cl.client.get_workers("t")[0].shards[0].offset
        assert cl.client.batch_remove(["filler"]) == [E.OK]
        assert cl.client.keystone().compact_pool("hbm0") >= 1
        assert cl.client.get_workers("t")[0].shards[0].offset != before, "compaction did not move the object"
        read_all(E.OK, "after compaction")
        for tier, expect in (("RAM_CPU", E.OK), ("NVME", E.NOT_IMPLEMENTED), ("RAM_GPU", E.OK)):
            assert cl.client.migrate("t", getattr(bb.StorageClass, tier)) == E.OK
            assert cl.client.get_workers("t")[0].shards[0].storage_class == getattr(bb.StorageClass, tier)
            read_all(expect, f"after a move to {tier}")
        # a corrupt copy in DRAM, read over PCIe: the same refresh
        assert cl.client.migrate("t", bb.StorageClass.RAM_CPU) == E.OK
        sh = cl.client.get_workers("t")[0].shards[0]
        store.flip(sh, 5)
        read_all(E.CHECKSUM_MISMATCH, "the only copy corrupt in DRAM")
        store.flip(sh, 5)
        read_all(E.OK, "DRAM restored")
    finally:
        cl.stop()
