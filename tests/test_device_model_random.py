"""Seeded random operation sequences through the client's device API on a GpuRankCluster with three tiers, against a
host model of the store.

The cluster has an HBM slab, a pinned shared-memory DRAM pool (which the fused kernels reach over PCIe) and an NVMe pool
(which device gets reach only through the host-staged path); ttl 0 and watermark 1.0, so nothing moves on its own.  Each
step draws a byte put (plain or strided source, 1-3 replicas, 1-2 workers per copy, any algorithm), an fp8 put (plain or
strided source), a byte get (whole, range or strided), an fp8 get (whole, range or strided), a tier move, a compaction
of the HBM pool, a corruption of one copy or of every copy of an object followed by gets of it, or a remove.  Batches
mix keys of different steps, tiers and algorithms; caller pointers are sometimes misaligned and some strided gaps are no
multiple of 16 bytes (8 elements).

The model predicts every item's error code from the documented rules, written out here: byte gets are staged, never
refused; an fp8 get is NOT_IMPLEMENTED when its virtual base is misaligned, when a multi-row slice has a gap that is no
multiple of 8 elements, or when the object sits on NVMe; CHECKSUM_MISMATCH only when every copy read is corrupt;
OBJECT_NOT_FOUND after a remove.  After every step it checks the result bytes and the guard bytes around them, every
copy's stored bytes and recorded digest (Store in test_device_path.py) and the client counters the step moves.

Models trusted: numpy slicing; bb.crc32c / bb.bbh64 / bb.xxh3t64 (checked in test_common.py against golden values,
_bbh64_numpy and python-xxhash); the exact MXFP8 model of test_mxfp8_exhaustive.py (checked there against torch)."""
import collections
import os

import numpy as np
import pytest
import torch

from test_device_path import Store, _counter, _ref
from test_mxfp8_exhaustive import model_pack, model_unpack, same_bits

pytestmark = pytest.mark.gpu

MiB = 1 << 20
GUARD = 0xA5
GUARD16 = 0x5A5A
T = 16384
ALGOS = ["NONE", "CRC32C", "BBH64", "XXH3"]
SEEDS = [3, 17]
STEPS = 150 + int(os.environ.get("BB_RANDOM_ROUNDS", "0")) * 10
OPS = ["put", "put_fp8", "get", "get_fp8", "migrate", "compact", "corrupt", "remove"]


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


class Obj:
    """The model of one object: its bytes (a packed object's packed bytes), algorithm, copies and tier."""

    def __init__(self, data, algo, copies, tier, x=None):
        self.data, self.algo, self.copies, self.tier, self.x = data, algo, copies, tier, x
        self.flips = set()  # (copy, shard) corrupt right now
        self.back = None if x is None else model_unpack(data, x.size)  # what an fp8 get returns

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
        reps, tier = 1, str(rng.choice(["RAM_GPU", "RAM_CPU"]))
        strided = rng.random() < 0.5
        self.what = f"fp8 put{' strided' if strided else ''} of {count}, {tier}"
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
            x = _bf16(rng, width * rows)
            buf = np.full((rows - 1) * pitch + width + 8, 0x7FC0, dtype=np.uint16)  # NaN in the gaps
            for i in range(rows):
                buf[i * pitch:i * pitch + width] = x[i * width:(i + 1) * width]
            srcs.append(torch.from_numpy(buf.view(np.int16)).cuda())
            shapes.append((width, pitch, rows))
            xs.append(x)
        cfg = _cfg(bb, "BBH64", reps, tier)
        ptrs = [s.data_ptr() for s in srcs]
        if strided:
            ecs = self.cl.client.batch_put_device_fp8_strided(keys, ptrs, [s[0] for s in shapes], [s[1] for s in shapes],
                                                              [s[2] for s in shapes], cfg, _stream())
        else:
            ecs = self.cl.client.batch_put_device_fp8(keys, ptrs, [x.size for x in xs], cfg, _stream())
        assert ecs == [bb.ErrorCode.OK] * count, f"{self.where()}: {ecs}"
        torch.cuda.synchronize()
        for k, x in zip(keys, xs):
            self.objs[k] = Obj(model_pack(x), "BBH64", reps, tier, x)

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
        items, o_ = [], 64
        for k in keys:
            o = self.objs.get(k)
            shape = ("range", 0, 64, 0, 1) if o is None else self._fp8_shape(o)
            # misaligned ranges and slices fail alone (NOT_IMPLEMENTED); a whole tensor's pointer is the engine's to check
            skew = int(rng.choice([1, 4])) if rng.random() < 0.2 and shape[0] != "whole" else 0
            region = (o_ + 7) // 8 * 8 + (shape[1] + skew) % 8  # element offset: virtual base aligned unless skewed
            items.append((k, o, shape, region, skew))
            o_ = region + shape[2] * shape[4] + 32
        out = torch.full((o_ + 64,), GUARD16, dtype=torch.int16, device="cuda")
        p = out.data_ptr()
        self.what = f"fp8 get of {len(keys)}"
        ecs = {}
        ref0, fo0 = self.counter("get_placement_refresh_total"), self.counter("replica_failover_total")
        for kind in ("whole", "range", "strided"):
            idx = [i for i, it in enumerate(items) if it[2][0] == kind]
            if not idx:
                continue
            ks = [items[i][0] for i in idx]
            ptrs = [p + 2 * items[i][3] for i in idx]
            ns = [items[i][1].x.size if items[i][1] is not None else 64 for i in idx]
            if kind == "whole":
                got = self.cl.client.batch_get_device_fp8(ks, ptrs, ns, _stream())
            elif kind == "range":
                got = self.cl.client.batch_get_device_fp8_range(ks, ptrs, ns, [items[i][2][1] for i in idx], [items[i][2][2] for i in idx], _stream())
            else:
                got = self.cl.client.batch_get_device_fp8_strided(ks, ptrs, ns, [items[i][2][1] for i in idx], [items[i][2][2] for i in idx],
                                                                  [items[i][2][3] for i in idx], [items[i][2][4] for i in idx], _stream())
            for i, ec in zip(idx, got):
                ecs[i] = ec
        torch.cuda.synchronize()
        want = np.full(out.numel(), GUARD16, dtype=np.uint16)
        written = np.zeros(out.numel(), dtype=bool)
        E = bb.ErrorCode
        mismatches = 0
        for i, (k, o, (kind, off, w, pitch, rows), region, skew) in enumerate(items):
            desc = f"{k} {kind} off={off} width={w} pitch={pitch} rows={rows} skew={skew}"
            if o is None:
                exp = E.OBJECT_NOT_FOUND
            else:
                desc += f" n={o.x.size} {o.tier} x{o.copies}"
                gap_bad = rows > 1 and w < pitch and (pitch - w) % 8 != 0
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
                want[region:region + el.size] = o.back[el]
                written[region:region + el.size] = True
                same_bits(out[region:region + el.size].cpu().numpy(), o.back[el], "bf16", self.where(i, desc))
            self.outcomes[str(exp).split(".")[-1]] += 1
            self.outcomes["fused"] += exp == E.OK
        got = out.cpu().numpy().view(np.uint16)
        bad = np.nonzero(~written & (got != GUARD16))[0]
        assert bad.size == 0, f"{self.where()}: {bad.size} elements written outside the results, first at {bad[:4].tolist()}"
        assert self.counter("get_placement_refresh_total") - ref0 == mismatches, f"{self.where()}: placement refreshes"
        self.outcomes["fail-over"] += self.counter("replica_failover_total") - fo0

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
        k = str(rng.choice(keys))
        o = self.objs[k]
        everyone = rng.random() < 0.5
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
            for _ in range(2):  # two gets: the shapes are drawn anew each time
                (self.get_fp8 if o.fp8 else self.get)([k] + others)
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
        weights = np.array([3, 2, 4, 4, 2, 1, 3, 1], dtype=float)
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
        for o in ("fused", "staged", "NOT_IMPLEMENTED", "CHECKSUM_MISMATCH", "fail-over", "OBJECT_NOT_FOUND"):
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
